// Tests of the host side of ICMP error translation (bng_nat_icmp_errors_enable): nat::ManagerConfig::
// EnableICMPErrorTranslation applied by nat::Manager::Start, shard::Router::NatICMPErrorsEnable reaching every shard,
// and Directory::SteerDownstream steering an ICMP error by the flow it quotes (bng_host.hpp, bng_shard.hpp).
// `test_nat_icmp_host cpu` needs no device: the NULL-context check and the steering.  `test_nat_icmp_host gpu`
// observes the flag through its effect: a subscriber's UDP frame is SNATed by nat44_egress, and a port-unreachable
// quoting it comes back through nat44_ingress addressed to the subscriber when translation is on, unchanged when off.
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

// A Destination Unreachable / port unreachable from a router at 192.0.2.1 to the quoted packet's source, quoting
// its IPv4 header and first 8 L4 bytes (q: the quoted packet's IPv4 header, as it left the NAT).  Frame length 70.
static void icmp_error(uint8_t *f, const uint8_t *q) {
    static const uint8_t router[4] = {192, 0, 2, 1};
    ipv4(f, router, q + 12, 1, 56);
    f[34] = 3, f[35] = 3;
    memcpy(f + 42, q, 28);
}

static int run(bng_ctx *c, const char *prog, std::vector<uint8_t> &frames, uint32_t n, uint32_t stride,
               std::vector<uint32_t> len, uint64_t now) {
    std::vector<uint8_t> verdict(n);
    bng_batch bt{};
    bt.pkts = frames.data(), bt.len = len.data(), bt.verdict = verdict.data(), bt.n = n, bt.stride = stride;
    bt.mem = BNG_MEM_HOST, bt.arena_bytes = (uint32_t)(frames.size() / 16), bt.now_ns = now;
    return bng_prog_run(c, bng_prog_id(c, prog), &bt);
}

// 100.64.0.<s>:40000 sends a UDP frame to 8.8.8.8:53 through nat44_egress; a port unreachable quoting the SNATed
// frame then goes through nat44_ingress.  Returns whether it came back to 100.64.0.<s>:40000.
static bool error_reaches_subscriber(bng_ctx *c, uint8_t s) {
    const uint8_t sub[4] = {100, 64, 0, s}, dns[4] = {8, 8, 8, 8};
    std::vector<uint8_t> up(64);
    ipv4(up.data(), sub, dns, 17, 50);
    put16(&up[34], 40000);
    put16(&up[36], 53);
    put16(&up[38], 30);
    CHECK(run(c, "nat44_egress", up, 1, 64, {64}, 1000000000ull) == 0);
    CHECK(memcmp(&up[26], sub, 4) != 0); // SNATed
    std::vector<uint8_t> down(128);
    icmp_error(down.data(), &up[14]);
    CHECK(run(c, "nat44_ingress", down, 1, 128, {70}, 2000000000ull) == 0);
    const bool outer = memcmp(&down[30], sub, 4) == 0, inner = memcmp(&down[54], sub, 4) == 0;
    const bool port = down[62] == (40000 >> 8) && down[63] == (40000 & 0xff);
    CHECK(outer == inner && inner == port);
    return outer && inner && port;
}

static bool launched(bng_ctx *c, const char *name) {
    std::vector<char> buf(1 << 16);
    int64_t n = bng_prof_read(c, buf.data(), buf.size());
    return n > 0 && std::string(buf.data(), (size_t)n).find(name) != std::string::npos;
}

static void test_null() {
    CHECK(bng_nat_icmp_errors_enable(nullptr, 1) == -EINVAL && bng_nat_icmp_errors_enable(nullptr, 0) == -EINVAL);
}

static const uint8_t k_pub[4] = {203, 0, 113, 5};

// A subscriber whose block (ports 1216-1279 of 203.0.113.5) is on shard 1, pinned there.
static void learn_pinned(shard::Directory &d) {
    const uint64_t mac = 0x020000000001ull;
    const uint8_t priv[4] = {100, 64, 0, 9};
    uint32_t pk, uk;
    memcpy(&pk, priv, 4);
    memcpy(&uk, k_pub, 4);
    d.Learn(mac, pk);
    d.Pin(mac, 1);
    d.AddBlock(uk, 1024 + 64 * 3, pk);
}

// A port unreachable quoting that subscriber's flow (public port / echo id 1220) of protocol proto; its own bytes 4-5
// are a next-hop MTU of 1500, which names no block.
static std::vector<uint8_t> error_to_pinned(int proto) {
    static const uint8_t remote[4] = {8, 8, 4, 4};
    std::vector<uint8_t> q(64), f(128);
    ipv4(q.data(), k_pub, remote, (uint8_t)proto, 48);
    if (proto == 1) {
        q[34] = 8;
        put16(&q[38], 1220); // the echo id: the public "port"
    } else {
        put16(&q[34], 1220);
        put16(&q[36], 53);
    }
    icmp_error(f.data(), &q[14]);
    put16(&f[38], 1500);
    return f;
}

// Directory only: errors quoting the pinned subscriber's TCP, UDP and ICMP echo flows.
static void test_steering() {
    shard::Directory d(2, 1024, 64);
    learn_pinned(d);
    for (int proto : {17, 6, 1}) {
        std::vector<uint8_t> f = error_to_pinned(proto);
        for (uint8_t type : {3, 11, 12}) {
            f[34] = type;
            d.SetICMPErrors(false);
            CHECK(d.SteerDownstream(f.data(), 70, 0) == 0); // as today: by bytes 4-5, nobody's
            d.SetICMPErrors(true);
            CHECK(d.SteerDownstream(f.data(), 70, 0) == 1); // by the quoted flow
            CHECK(d.SteerDownstream(f.data(), proto == 1 ? 67 : 65, 0) == 0); // the quoted port / id not present
        }
        f[34] = 0; // an echo reply is steered by its id as before
        put16(&f[38], 1230);
        CHECK(d.SteerDownstream(f.data(), 70, 0) == 1);
        put16(&f[38], 1500);
        CHECK(d.SteerDownstream(f.data(), 70, 0) == 0);
        f[34] = 3;
        f[54] ^= 1; // quoted source is not the outer destination: not translatable, to fallback
        CHECK(d.SteerDownstream(f.data(), 70, 0) == 0);
    }
    // every length up to the whole frame, each held in a buffer of exactly that many bytes: the quoted flow steers
    // only once its port (TCP/UDP, through byte 65) or id (ICMP, through 67) is present, and nothing past `len` is read
    for (int proto : {17, 6, 1}) {
        const std::vector<uint8_t> f = error_to_pinned(proto);
        const uint32_t need = proto == 1 ? 68 : 66;
        for (uint32_t len = 0; len <= 70; len++) {
            std::unique_ptr<uint8_t[]> exact(new uint8_t[len ? len : 1]);
            memcpy(exact.get(), f.data(), len);
            CHECK(d.SteerDownstream(exact.get(), len, 0) == (len >= need ? 1u : 0u));
        }
    }
}

static void test_gpu_manager() {
    for (bool on : {false, true}) {
        auto be = open_ctx(0, 1);
        if (!be->ctx) return;
        nat::ManagerConfig cfg;
        cfg.Interface = "eth0", cfg.Backend_ = be, cfg.PortsPerSubscriber = 64, cfg.EnableICMPErrorTranslation = on;
        auto m = nat::Manager::NewManager(cfg);
        CHECK(m.ok());
        CHECK(!(*m)->Start());
        CHECK(!(*m)->AddPublicIP(IPv4(203, 0, 113, 1)));
        for (uint8_t s : {1, 2}) {
            CHECK((*m)->AllocateNAT(IPv4(100, 64, 0, s)).ok());
            CHECK(error_reaches_subscriber(be->ctx, s) == on);
        }
    }
}

static void test_gpu_router() {
    auto dir = std::make_shared<shard::Directory>(2, 1024, 64);
    std::vector<std::shared_ptr<Backend>> shards = {open_ctx(0, 2), open_ctx(1, 2)};
    if (!shards[0]->ctx || !shards[1]->ctx) return;
    shard::Router r(shards, dir);
    std::vector<uint8_t> f(64);
    auto probe = [&](const char *name) {
        bool all = true;
        for (auto &s : shards) {
            CHECK(bng_prof_enable(s->ctx, 1) == 0);
            CHECK(run(s->ctx, "nat44_ingress", f, 1, 64, {64}, 1000000000ull) == 0);
            all = all && launched(s->ctx, name);
            CHECK(bng_prof_enable(s->ctx, 0) == 0);
        }
        return all;
    };
    CHECK(probe("k_nat_ingress ") && !probe("k_nat_ingress<icmperr>")); // off by default
    learn_pinned(*dir);
    const std::vector<uint8_t> e = error_to_pinned(17);
    CHECK(dir->SteerDownstream(e.data(), 70, 0) == 0);
    CHECK(r.NatICMPErrorsEnable(true) == 0);
    CHECK(probe("k_nat_ingress<icmperr>"));
    CHECK(dir->SteerDownstream(e.data(), 70, 0) == 1); // the Router told its Directory
    CHECK(r.NatICMPErrorsEnable(false) == 0);
    CHECK(!probe("k_nat_ingress<icmperr>"));
    CHECK(dir->SteerDownstream(e.data(), 70, 0) == 0);
}

// One context against two shards behind a Router with the flag on: every subscriber's flows are made upstream on its
// shard (SteerUpstream), and replies and ICMP errors quoting those flows, of every length from 34 to 92 bytes and of
// every kind the rule passes, are steered by Directory::SteerDownstream.  The shards' frames, verdicts and NAT counters
// add up to the one context's.
static void test_gpu_sharded() {
    const uint32_t world = 2, n_subs = 16;
    auto dir = std::make_shared<shard::Directory>(world, 1024, 64);
    std::vector<std::shared_ptr<Backend>> shards = {open_ctx(0, world), open_ctx(1, world)};
    auto whole = open_ctx(0, 1);
    if (!shards[0]->ctx || !shards[1]->ctx || !whole->ctx) return;
    shard::Router r(shards, dir);
    CHECK(r.NatICMPErrorsEnable(true) == 0);
    CHECK(bng_nat_icmp_errors_enable(whole->ctx, 1) == 0);
    // the same blocks everywhere: every context's manager allocates every subscriber, in the same order
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
    // upstream: by MAC to the shards, everything to the one context
    std::vector<uint8_t> snat = up;
    CHECK(run(whole->ctx, "nat44_egress", snat, n_up, 64, std::vector<uint32_t>(n_up, 64), 1000000000ull) == 0);
    uint32_t seen[2] = {0, 0};
    for (uint32_t i = 0; i < n_up; i++) {
        std::vector<uint8_t> one(up.begin() + i * 64, up.begin() + (i + 1) * 64);
        const uint32_t k = dir->SteerUpstream(one.data(), 64);
        seen[k]++;
        CHECK(run(shards[k]->ctx, "nat44_egress", one, 1, 64, {64}, 1000000000ull) == 0);
        CHECK(memcmp(one.data(), &snat[i * 64], 64) == 0);
    }
    CHECK(seen[0] > 0 && seen[1] > 0);
    // downstream: a reply to every flow, and errors quoting it of every length, type and kind
    std::vector<uint8_t> down;
    std::vector<uint32_t> lens;
    auto add = [&](const uint8_t *f, uint32_t len) {
        down.insert(down.end(), f, f + 128);
        lens.push_back(len);
    };
    for (uint32_t i = 0; i < n_up; i++) {
        const uint8_t *q = &snat[i * 64];
        uint8_t f[128] = {0};
        memcpy(f, q, 64);
        memcpy(f + 26, q + 30, 4), memcpy(f + 30, q + 26, 4);
        if (q[23] == 1)
            f[34] = 0;
        else
            memcpy(f + 34, q + 36, 2), memcpy(f + 36, q + 34, 2);
        add(f, 64);
        for (uint32_t len = 34 + i % 3; len <= 92; len += 3) {
            memset(f, 0, sizeof f);
            icmp_error(f, q + 14);
            memcpy(f + 42, q + 14, 50); // the whole quoted packet
            f[34] = (uint8_t)(len % 2 ? 11 : (len % 3 ? 3 : 12));
            if (len % 7 == 0) f[30] ^= 1;      // not addressed to the quoted source
            if (len % 11 == 0) f[65] ^= 0x40;  // a quoted port no flow has
            add(f, len);
        }
    }
    const uint32_t n = (uint32_t)lens.size();
    std::vector<uint8_t> one = down;
    CHECK(run(whole->ctx, "nat44_ingress", one, n, 128, lens, 2000000000ull) == 0);
    uint32_t to[2] = {0, 0};
    for (uint32_t i = 0; i < n; i++) {
        const std::vector<uint8_t> exact(down.begin() + i * 128, down.begin() + i * 128 + lens[i]); // len bytes
        const uint32_t k = dir->SteerDownstream(exact.data(), lens[i], 0);
        to[k]++;
        std::vector<uint8_t> f(down.begin() + i * 128, down.begin() + (i + 1) * 128); // the whole slot, as in `one`
        CHECK(run(shards[k]->ctx, "nat44_ingress", f, 1, 128, {lens[i]}, 2000000000ull) == 0);
        CHECK(memcmp(f.data(), &one[i * 128], 128) == 0);
    }
    CHECK(to[0] > 0 && to[1] > 0);
    uint64_t st[3][13];
    for (int c = 0; c < 3; c++) {
        uint32_t key = 0;
        CHECK(bng_map_lookup(all[c]->ctx, bng_map_id(all[c]->ctx, "nat_stats_map"), &key, st[c]) == 0);
    }
    for (int j = 0; j < 13; j++) CHECK(st[0][j] + st[1][j] == st[2][j]);
    CHECK(st[2][1] > n_up); // packets_dnat: the replies and many errors
}

int main(int argc, char **argv) {
    std::string mode = argc > 1 ? argv[1] : "cpu";
    test_null();
    test_steering();
    if (mode == "gpu") {
        test_gpu_manager();
        test_gpu_router();
        test_gpu_sharded();
    }
    printf("%d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
