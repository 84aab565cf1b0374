// The section framing of the library's state blobs (include/bng_b200.h): bng_snapshot, bng_delta_export and
// bng_sub_export.  After a format's own header, each section is a 64-byte header, then its keys, then its values; a
// delta section lists its deleted keys (as many as `pad` says) ahead of the keys.  Host-only: no CUDA, no bng_ctx.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace blob {

const char kSnapMagic[8] = {'B', 'N', 'G', 'S', 'N', 'A', 'P', '2'};
const char kDeltaMagic[8] = {'B', 'N', 'G', 'D', 'E', 'L', 'T', '1'};
const char kMoveMagic[8] = {'B', 'N', 'G', 'M', 'O', 'V', 'E', '1'};

struct DeltaHdr {
    char magic[8];
    uint64_t stream, seq_from, seq_to;
    uint32_t flags, sections;
};

struct SectionHdr {
    char name[40];
    uint32_t kind, key_size, value_size, pad; // pad: the deleted keys of a delta section
    uint64_t count;
};
static_assert(sizeof(DeltaHdr) == 40 && sizeof(SectionHdr) == 64, "the framing of include/bng_b200.h");

// The record sections.  No map has these names, so a library without the feature steps over them.
// Accounting records: (address, struct bng_acct) pairs; a context that never allocated records writes none.
const char kAcct[] = "subscriber_acct";
const uint32_t kAcctKind = 5;
// Interception targets: (address, target id) pairs, by address.  The intercepted records are not state and stay out.
const char kLi[] = "li_targets";
const uint32_t kLiKind = 6;
// Idle timeouts: (address, uint32 timeout_s) pairs, by address.  The clocks are not state (another node's clock, or
// this one's minutes ago, says nothing about activity now).
const char kIdle[] = "subscriber_idle";
const uint32_t kIdleKind = 7;
// Whole idle records, (address, struct bng_idle), in hand-over blobs only: a name of their own, so that restore and
// delta apply, which take only timeouts under kIdle, step over them.
const char kIdleRec[] = "subscriber_idle_rec";
const uint32_t kIdleRecKind = 8;

// Appends sections after a header of hdr_len bytes that the caller fills in, with the count of sections where its
// format keeps it.
struct Writer {
    std::vector<uint8_t> out;
    uint64_t sections = 0;

    explicit Writer(size_t hdr_len) : out(hdr_len) {}

    // a section header; the caller appends n_del deleted keys, then count keys, then count values
    void header(const char *name, uint32_t kind, uint32_t key_size, uint32_t value_size, uint64_t count, uint32_t n_del = 0) {
        SectionHdr h{};
        snprintf(h.name, sizeof(h.name), "%s", name);
        h.kind = kind, h.key_size = key_size, h.value_size = value_size, h.pad = n_del, h.count = count;
        append(&h, sizeof(h));
        sections++;
    }
    void append(const void *p, size_t n) { out.insert(out.end(), (const uint8_t *)p, (const uint8_t *)p + n); }
    void section(const char *name, uint32_t kind, uint32_t key_size, uint32_t value_size, uint64_t count, const void *keys,
                 const void *vals) {
        header(name, kind, key_size, value_size, count);
        append(keys, count * key_size);
        append(vals, count * value_size);
    }
    // an (address, u32) section
    void pairs(const char *name, uint32_t kind, const std::vector<uint32_t> &addrs, const std::vector<uint32_t> &vals) {
        section(name, kind, 4, 4, addrs.size(), addrs.data(), vals.data());
    }
};

struct Section {
    SectionHdr h;   // name NUL-terminated
    uint64_t n_del; // h.pad when read with_del, else 0
    const uint8_t *dels, *keys, *vals;
};

// Reads n sections from [p, end) into out.  with_del: pad counts deleted keys (deltas); exact_end: no byte may follow
// the last section.  Every size is checked against what is left without overflow.  False, with err saying why, on a
// blob that does not hold its sections.
inline bool read_sections(const uint8_t *p, const uint8_t *end, uint64_t n, bool with_del, bool exact_end,
                          std::vector<Section> &out, std::string &err) {
    char msg[96];
    for (uint64_t k = 0; k < n; k++) {
        Section s{};
        if ((uint64_t)(end - p) < sizeof(SectionHdr)) {
            snprintf(msg, sizeof(msg), "section %llu of %llu is truncated", (unsigned long long)k, (unsigned long long)n);
            err = msg;
            return false;
        }
        memcpy(&s.h, p, sizeof(s.h));
        p += sizeof(s.h);
        s.h.name[sizeof(s.h.name) - 1] = 0;
        s.n_del = with_del ? s.h.pad : 0;
        const uint64_t left = (uint64_t)(end - p), del_bytes = s.n_del * s.h.key_size; // < 2^64: two 32-bit factors
        const uint64_t per = (uint64_t)s.h.key_size + s.h.value_size;
        if (del_bytes > left || (per && s.h.count > (left - del_bytes) / per)) {
            err = std::string(s.h.name) + " is truncated";
            return false;
        }
        s.dels = p;
        s.keys = p + del_bytes;
        s.vals = s.keys + s.h.count * s.h.key_size;
        p = s.vals + s.h.count * s.h.value_size;
        out.push_back(s);
    }
    if (exact_end && p != end) {
        snprintf(msg, sizeof(msg), "%llu bytes after the last section", (unsigned long long)(end - p));
        err = msg;
        return false;
    }
    return true;
}

} // namespace blob
