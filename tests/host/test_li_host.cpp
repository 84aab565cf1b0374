// intercept::ParseCC / PumpRecords on synthetic bng_li_record records (no GPU needed), and the record layout.
//   test_li_host layout   prints the header's field offsets for the Python side to compare against layouts.py
//   test_li_host cpu      the parse checks
#include <cstdio>
#include <cstdlib>
#include <string>

#include "../../bng_b200/host/bng_host.hpp"

using namespace bng;

static int failures = 0;
#define CHECK(c)                                                             \
    do {                                                                     \
        if (!(c)) {                                                          \
            fprintf(stderr, "%s:%d: CHECK failed: %s\n", __FILE__, __LINE__, #c); \
            failures++;                                                      \
        }                                                                    \
    } while (0)

static_assert(sizeof(bng_li_record) == 64, "bng_li_record is 64 bytes");

// one record: header + frame bytes (Ethernet, IPv4 with ihl words, L4), rec_size bytes
static std::vector<uint8_t> make_record(uint32_t rec_size, uint32_t target, uint8_t dir, uint8_t proto, uint32_t ihl,
                                        uint32_t cap_len, const std::vector<uint8_t> &l4) {
    std::vector<uint8_t> r(rec_size, 0);
    bng_li_record h{};
    h.ts_ns = 123456789;
    h.batch = 3;
    h.frame = 17;
    h.target_id = target;
    h.addr = 0x0A004064;
    h.wire_len = 1000;
    h.cap_len = cap_len;
    h.dir = dir;
    h.verdict = BNG_TC_ACT_OK;
    h.prog = 7;
    memcpy(r.data(), &h, sizeof(h));
    std::vector<uint8_t> f(14 + 4 * ihl + l4.size(), 0);
    f[12] = 0x08;
    f[14] = (uint8_t)(0x40 | ihl);
    f[23] = proto;
    const uint8_t src[4] = {100, 64, 0, 10}, dst[4] = {8, 8, 4, 4};
    memcpy(&f[26], src, 4);
    memcpy(&f[30], dst, 4);
    for (uint32_t k = 34; k < 14 + 4 * ihl; k++) f[k] = 0x01; // IPv4 options: NOPs
    memcpy(&f[14 + 4 * ihl], l4.data(), l4.size());
    memcpy(r.data() + 64, f.data(), std::min<size_t>(f.size(), cap_len));
    return r;
}

static intercept::CC parse(const std::vector<uint8_t> &r) {
    intercept::CC cc;
    intercept::ParseCC(r.data(), &cc);
    return cc;
}

int main(int argc, char **argv) {
    const std::string mode = argc > 1 ? argv[1] : "cpu";
    if (mode == "layout") {
        printf("size %zu\n", sizeof(bng_li_record));
#define OFF(f) printf(#f " %zu\n", offsetof(bng_li_record, f))
        OFF(ts_ns); OFF(batch); OFF(frame); OFF(target_id); OFF(addr); OFF(wire_len); OFF(cap_len); OFF(dir); OFF(verdict);
        OFF(prog); OFF(pad);
        return 0;
    }
    const uint32_t rs = 64 + 128;
    const std::vector<uint8_t> tcp = {0x1f, 0x90, 0x00, 0x50, 0, 0, 0, 0, 0, 0, 0, 0, 0x50, 0x10, 0, 0, 0, 0, 0, 0};
    const std::vector<uint8_t> udp = {0x13, 0x88, 0x00, 0x35, 0x00, 0x10, 0, 0};
    const std::vector<uint8_t> echo = {8, 0, 0, 0, 0x12, 0x34, 0x00, 0x01};
    const std::vector<uint8_t> unreach = {3, 1, 0, 0, 0x12, 0x34, 0x00, 0x01};
    { // TCP, ihl 5
        auto cc = parse(make_record(rs, 1, BNG_LI_UPLINK, 6, 5, 54, tcp));
        CHECK(cc.direction == intercept::Direction::Uplink && cc.protocol == 6);
        CHECK(cc.src == IPv4(100, 64, 0, 10) && cc.dst == IPv4(8, 8, 4, 4));
        CHECK(cc.src_port == 8080 && cc.dst_port == 80);
        CHECK(cc.payload.size() == 40 && cc.payload[0] == 0x45 && cc.rec.frame == 17 && cc.rec.batch == 3);
    }
    { // UDP behind 8 bytes of IPv4 options
        auto cc = parse(make_record(rs, 1, BNG_LI_DOWNLINK, 17, 7, 14 + 28 + 8, udp));
        CHECK(cc.direction == intercept::Direction::Downlink && cc.src_port == 5000 && cc.dst_port == 53);
        CHECK(cc.payload.size() == 36 && cc.payload[0] == 0x47);
    }
    { // ICMP echo: the id is the subscriber-side port
        auto up = parse(make_record(rs, 1, BNG_LI_UPLINK, 1, 5, 42, echo));
        CHECK(up.src_port == 0x1234 && up.dst_port == 0);
        auto down = parse(make_record(rs, 1, BNG_LI_DOWNLINK, 1, 5, 42, echo));
        CHECK(down.src_port == 0 && down.dst_port == 0x1234);
        auto other = parse(make_record(rs, 1, BNG_LI_UPLINK, 1, 5, 42, unreach));
        CHECK(other.src_port == 0 && other.dst_port == 0);
        auto gre = parse(make_record(rs, 1, BNG_LI_UPLINK, 47, 5, 42, udp));
        CHECK(gre.protocol == 47 && gre.src_port == 0 && gre.dst_port == 0);
    }
    { // captures cut short
        auto ports_cut = parse(make_record(rs, 1, BNG_LI_UPLINK, 6, 5, 36, tcp)); // source port only
        CHECK(ports_cut.src_port == 0 && ports_cut.dst_port == 0 && ports_cut.dst == IPv4(8, 8, 4, 4));
        auto opts_cut = parse(make_record(rs, 1, BNG_LI_UPLINK, 17, 7, 44, udp)); // ends inside the UDP header
        CHECK(opts_cut.src_port == 0 && opts_cut.dst_port == 0);
        intercept::CC cc;
        auto r = make_record(rs, 1, BNG_LI_UPLINK, 17, 5, 31, udp); // source address only
        CHECK(!intercept::ParseCC(r.data(), &cc));
        CHECK(cc.src == IPv4(100, 64, 0, 10) && cc.dst == IPv4(0, 0, 0, 0) && cc.payload.size() == 17);
    }
    { // the resolver: records of an unknown target are skipped
        std::vector<uint8_t> all;
        for (uint32_t t : {1u, 2u, 1u, 3u}) {
            auto r = make_record(rs, t, BNG_LI_UPLINK, 17, 5, 42, udp);
            all.insert(all.end(), r.begin(), r.end());
        }
        std::vector<std::string> seen;
        intercept::Resolver<std::string> resolve = [](uint32_t id) -> std::optional<std::string> {
            if (id == 2) return std::nullopt; // an IRI-only warrant
            return "warrant-" + std::to_string(id);
        };
        intercept::Sink<std::string> sink = [&](const std::string &w, const intercept::CC &cc) {
            seen.push_back(w + ":" + std::to_string(cc.src_port));
        };
        const uint64_t n = intercept::PumpRecords<std::string>(all.data(), 4, rs, resolve, sink);
        CHECK(n == 3);
        CHECK((seen == std::vector<std::string>{"warrant-1:5000", "warrant-1:5000", "warrant-3:5000"}));
    }
    if (failures) {
        fprintf(stderr, "%d check(s) failed\n", failures);
        return 1;
    }
    printf("ok\n");
    return 0;
}
