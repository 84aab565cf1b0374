// The section framing of the state blobs (bng_b200/csrc/blob.hpp) on the host alone: the writer's bytes against a
// section spelled out from include/bng_b200.h, round trips with and without deleted keys, and the reader's refusals.
#include <cstdio>
#include <cstdlib>

#include "../../bng_b200/csrc/blob.hpp"

static int failures = 0;
#define CHECK(c)                                                             \
    do {                                                                     \
        if (!(c)) {                                                          \
            fprintf(stderr, "%s:%d: CHECK failed: %s\n", __FILE__, __LINE__, #c); \
            failures++;                                                      \
        }                                                                    \
    } while (0)

using Bytes = std::vector<uint8_t>;

static void put_le(Bytes &b, uint64_t v, int n) {
    for (int i = 0; i < n; i++) b.push_back((uint8_t)(v >> (8 * i)));
}

// a section header as include/bng_b200.h describes it: char name[40]; u32 kind, key_size, value_size, pad; u64 count
static void spell_header(Bytes &b, const char *name, uint32_t kind, uint32_t ks, uint32_t vs, uint32_t pad, uint64_t count) {
    const size_t at = b.size();
    b.resize(at + 40, 0);
    memcpy(&b[at], name, strlen(name));
    put_le(b, kind, 4), put_le(b, ks, 4), put_le(b, vs, 4), put_le(b, pad, 4), put_le(b, count, 8);
}

static bool read(const Bytes &b, size_t hdr, uint64_t n, bool with_del, bool exact_end, std::vector<blob::Section> &out) {
    std::string err;
    out.clear();
    const bool ok = blob::read_sections(b.data() + hdr, b.data() + b.size(), n, with_del, exact_end, out, err);
    CHECK(ok == err.empty());
    return ok;
}

static bool refused(const Bytes &b, size_t hdr, uint64_t n, bool with_del, bool exact_end) {
    std::vector<blob::Section> out;
    return !read(b, hdr, n, with_del, exact_end, out);
}

static void exact_bytes() {
    blob::Writer w(16);
    w.pairs(blob::kLi, blob::kLiKind, {0x0A000001, 0x0A000002}, {7, 8});
    const uint16_t keys[3] = {1, 2, 3};
    const uint8_t vals[3] = {9, 8, 7};
    w.header("m", 1, 2, 1, 3, 5);
    w.append(keys, sizeof(keys));
    w.append(vals, sizeof(vals));
    Bytes want(16, 0);
    spell_header(want, "li_targets", 6, 4, 4, 0, 2);
    put_le(want, 0x0A000001, 4), put_le(want, 0x0A000002, 4), put_le(want, 7, 4), put_le(want, 8, 4);
    spell_header(want, "m", 1, 2, 1, 5, 3);
    put_le(want, 1, 2), put_le(want, 2, 2), put_le(want, 3, 2), put_le(want, 0x070809, 3);
    CHECK(w.sections == 2);
    CHECK(w.out == want);
    // a name of 40 or more characters keeps its NUL
    blob::Writer l(0);
    l.header("0123456789012345678901234567890123456789xyz", 1, 0, 0, 0);
    CHECK(l.out.size() == 64 && l.out[39] == 0 && l.out[38] == '8');
}

static void round_trips() {
    const uint32_t del[2] = {11, 12}, keys[3] = {1, 2, 3};
    const uint64_t vals[3] = {100, 200, 300};
    // with deleted keys (a delta)
    blob::Writer d(sizeof(blob::DeltaHdr));
    d.header("nat_sessions", 1, 4, 8, 3, 2);
    d.append(del, sizeof(del)), d.append(keys, sizeof(keys)), d.append(vals, sizeof(vals));
    d.header("empty", 2, 4, 4, 0, 0);
    d.pairs(blob::kIdle, blob::kIdleKind, {5}, {300});
    std::vector<blob::Section> s;
    CHECK(read(d.out, sizeof(blob::DeltaHdr), d.sections, true, true, s) && s.size() == 3);
    if (s.size() == 3) {
        CHECK(!strcmp(s[0].h.name, "nat_sessions") && s[0].h.kind == 1 && s[0].n_del == 2 && s[0].h.count == 3);
        CHECK(!memcmp(s[0].dels, del, sizeof(del)) && !memcmp(s[0].keys, keys, sizeof(keys)) && !memcmp(s[0].vals, vals, sizeof(vals)));
        CHECK(!strcmp(s[1].h.name, "empty") && s[1].h.count == 0 && s[1].n_del == 0);
        uint32_t a, t;
        memcpy(&a, s[2].keys, 4), memcpy(&t, s[2].vals, 4);
        CHECK(!strcmp(s[2].h.name, "subscriber_idle") && s[2].h.kind == 7 && a == 5 && t == 300);
    }
    // without (a snapshot or hand-over blob): pad is not read, however it is set
    blob::Writer w(16);
    w.section("subscriber_nat", 1, 4, 8, 3, keys, vals);
    w.pairs(blob::kAcct, blob::kAcctKind, {}, {});
    w.out[16 + 52] = 0xEE; // the first section's pad
    CHECK(read(w.out, 16, w.sections, false, true, s) && s.size() == 2);
    if (s.size() == 2) {
        CHECK(s[0].n_del == 0 && s[0].h.pad == 0xEE && s[0].keys == w.out.data() + 16 + 64);
        CHECK(!memcmp(s[0].keys, keys, sizeof(keys)) && !memcmp(s[0].vals, vals, sizeof(vals)));
        CHECK(!strcmp(s[1].h.name, "subscriber_acct") && s[1].h.count == 0 && s[1].vals == w.out.data() + w.out.size());
    }
}

static void refusals() {
    const uint32_t keys[2] = {1, 2}, vals[2] = {3, 4};
    blob::Writer w(16);
    w.section("a", 1, 4, 4, 2, keys, vals);
    w.section("b", 1, 4, 4, 2, keys, vals);
    const Bytes &b = w.out;
    CHECK(!refused(b, 16, 2, false, true));
    CHECK(refused(b, 16, 3, false, false)); // a section more than there is
    for (size_t cut = 16 + 80 + 1; cut < b.size(); cut++) { // the second header, then its body, cut short
        Bytes t(b.begin(), b.begin() + cut);
        CHECK(refused(t, 16, 2, false, false));
    }
    // count * (key_size + value_size) that wraps to 0: 2^61 * 8
    Bytes wrap(b);
    spell_header(wrap, "subscriber_idle", 7, 4, 4, 0, 1ull << 61);
    CHECK(refused(wrap, 16, 3, false, false));
    Bytes wrap2(b); // and to 8 bytes, which follow
    spell_header(wrap2, "c", 1, 4, 4, 0, (1ull << 61) + 1);
    put_le(wrap2, 0, 8);
    CHECK(refused(wrap2, 16, 3, false, false));
    // n_del * key_size + count * (key_size + value_size) that wraps to 1 byte, which follows
    Bytes del(b);
    spell_header(del, "d", 1, 0xFFFFFFFFu, 1, 0xFFFFFFFFu, 2);
    del.push_back(0);
    CHECK(refused(del, 16, 3, true, false));
    CHECK(refused(del, 16, 3, false, false)); // without deleted keys the count alone does not fit either
    // trailing bytes: refused only with exact_end
    Bytes tail(b);
    tail.push_back(0);
    CHECK(refused(tail, 16, 2, false, true));
    CHECK(!refused(tail, 16, 2, false, false));
}

int main() {
    exact_bytes();
    round_trips();
    refusals();
    if (failures) {
        fprintf(stderr, "%d failures\n", failures);
        return 1;
    }
    printf("blob framing ok\n");
    return 0;
}
