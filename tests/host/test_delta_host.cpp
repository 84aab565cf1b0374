// ha::ParseDelta and ha::DataplaneSync without a GPU.
//   test_delta_host parse FILE   prints the header and one line per section of a delta blob, for the Python side to
//                                compare with bng_b200.layouts.parse_delta
//   test_delta_host cpu          DataplaneSync's sequence handling against a model of the library's rule
#include <cstdio>
#include <cstdlib>
#include <deque>
#include <string>

#include "../../bng_b200/host/bng_host.hpp"

using namespace bng;

static int failures = 0;
#define CHECK(c)                                                                  \
    do {                                                                          \
        if (!(c)) {                                                               \
            fprintf(stderr, "%s:%d: CHECK failed: %s\n", __FILE__, __LINE__, #c); \
            failures++;                                                           \
        }                                                                         \
    } while (0)

static uint64_t sum(const uint8_t *p, uint64_t n) {
    uint64_t s = 0;
    for (uint64_t i = 0; i < n; i++) s = s * 131 + p[i];
    return s;
}

static int parse(const char *path) {
    FILE *f = fopen(path, "rb");
    if (!f) return 2;
    std::vector<uint8_t> b;
    int ch;
    while ((ch = fgetc(f)) != EOF) b.push_back((uint8_t)ch);
    fclose(f);
    ha::DeltaHeader h{};
    std::string lines;
    bool ok = ha::ParseDelta(b.data(), b.size(), &h, [&](const ha::DeltaSection &s) {
        char line[256];
        snprintf(line, sizeof(line), "%s %u %u %u %u %llu %llu %llu\n", s.name.c_str(), s.kind, s.key_size, s.value_size, s.n_del,
                 (unsigned long long)s.n_up, (unsigned long long)sum(s.del_keys, (uint64_t)s.n_del * s.key_size),
                 (unsigned long long)sum(s.up_keys, s.n_up * s.key_size + s.n_up * s.value_size));
        lines += line;
    });
    if (!ok) {
        printf("invalid\n");
        return 0;
    }
    printf("header %llu %llu %llu %u %u\n%s", (unsigned long long)h.stream_id, (unsigned long long)h.seq_from,
           (unsigned long long)h.seq_to, h.flags, h.sections, lines.c_str());
    return 0;
}

// The library's rule, restated: exports carry (stream, seq_from, seq_to); an apply accepts FULL, or the next in sequence.
struct Model {
    uint64_t stream = 0x1234, seq = 0, a_stream = 0, a_seq = 0;
    bool first = true;
    size_t size = 100000; // bytes of every delta: larger than DataplaneSync's first buffer
    int exports = 0, enospc = 0;
    std::vector<uint8_t> Blob(uint32_t flags) {
        std::vector<uint8_t> b(size, 0);
        ha::DeltaHeader h{};
        memcpy(h.magic, "BNGDELT1", 8);
        h.stream_id = stream, h.seq_from = seq, h.seq_to = seq + 1, h.flags = flags;
        memcpy(b.data(), &h, sizeof(h));
        b.resize(sizeof(h)); // no sections
        return b;
    }
    ha::DeltaOps Ops() {
        ha::DeltaOps o;
        o.Export = [this](uint64_t, uint32_t flags, void *buf, uint64_t cap, uint64_t *len) {
            if (first) flags |= BNG_DELTA_FULL;
            auto b = Blob(flags);
            *len = b.size() + size; // a body the test does not look at
            if (cap < *len) {
                enospc++;
                return -ENOSPC;
            }
            memset(buf, 0, *len);
            memcpy(buf, b.data(), b.size());
            seq++, first = false, exports++;
            return 0;
        };
        o.Apply = [this](const void *buf, uint64_t) {
            ha::DeltaHeader h;
            memcpy(&h, buf, sizeof(h));
            if (!(h.flags & BNG_DELTA_FULL) && (h.stream_id != a_stream || h.seq_from != a_seq)) return -ESTALE;
            a_stream = h.stream_id, a_seq = h.seq_to;
            return 0;
        };
        return o;
    }
};

static void seq_handling() {
    Model m;
    std::deque<std::vector<uint8_t>> wire;
    ha::DataplaneSync *active_p = nullptr;
    ha::DataplaneSync active(m.Ops());
    ha::DataplaneSync standby(m.Ops(), [&] { active_p->RequestFull(); });
    active_p = &active;
    auto send = [&](bool full = false) {
        auto r = active.Export(0, full);
        CHECK(r.ok());
        if (!r.ok()) return;
        r->resize(sizeof(ha::DeltaHeader)); // the model's body is padding; the header alone is a delta without sections
        wire.push_back(*r);
    };
    auto deliver = [&]() {
        auto b = wire.front();
        wire.pop_front();
        return standby.Apply(b.data(), b.size());
    };
    send();
    CHECK(m.enospc == 1 && m.exports == 1); // the first buffer was too small: grown and repeated once
    CHECK(!deliver() && standby.Applied() == 1);
    send();
    CHECK(m.enospc == 1); // the grown buffer is kept
    CHECK(!deliver() && standby.Applied() == 2);
    // a lost delta: the next one is refused, FULL is requested once, refused deltas do not ask again
    send();
    wire.pop_front();
    send();
    CHECK((bool)deliver() && standby.FullRequests() == 1 && active.FullPending());
    send(); // FULL, since the peer asked
    CHECK(!active.FullPending());
    {
        ha::DeltaHeader h;
        memcpy(&h, wire.back().data(), sizeof(h));
        CHECK(h.flags & BNG_DELTA_FULL);
    }
    CHECK(!deliver() && standby.Applied() == 5);
    send();
    CHECK(!deliver() && standby.Applied() == 6 && standby.FullRequests() == 1);
    // a foreign stream (the active node restarted tracking): both deltas already on the wire are refused, FULL is
    // asked for once, and the active's next delta is FULL
    m.stream = 0x9999;
    send();
    send();
    CHECK((bool)deliver() && standby.FullRequests() == 2);
    CHECK((bool)deliver() && standby.FullRequests() == 2);
    send();
    CHECK(!deliver() && standby.Applied() == 9);
    send(true); // FullSyncInterval
    CHECK(!deliver() && standby.Applied() == 10 && standby.FullRequests() == 2);
}

int main(int argc, char **argv) {
    if (argc > 2 && !strcmp(argv[1], "parse")) return parse(argv[2]);
    if (argc > 1 && !strcmp(argv[1], "cpu")) {
        seq_handling();
        if (failures) fprintf(stderr, "%d failures\n", failures);
        else printf("ok\n");
        return failures ? 1 : 0;
    }
    fprintf(stderr, "usage: %s parse FILE | cpu\n", argv[0]);
    return 2;
}
