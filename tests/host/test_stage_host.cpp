// The control-plane staging (bng_b200/csrc/stage.hpp) against a fake runtime (fake_cuda/cuda_runtime_api.h), whose
// "device" memory is host memory: region offsets, chunk boundaries, one copy each way and one synchronisation per chunk,
// where a failure stops the loop, and the counted dump's min(count, cap).
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../bng_b200/csrc/stage.hpp"

static int failures = 0;
#define CHECK(c)                                                             \
    do {                                                                     \
        if (!(c)) {                                                          \
            fprintf(stderr, "%s:%d: CHECK failed: %s\n", __FILE__, __LINE__, #c); \
            failures++;                                                      \
        }                                                                    \
    } while (0)

static fake::State &S = fake::st();
static const uint64_t CHUNK = 8;

static void layout() {
    stage::Layout l;
    CHECK(l.take(10) == 0 && l.end == 10);
    CHECK(l.take(1) == 256 && l.end == 257);
    CHECK(l.take(0) == 512 && l.end == 512);
    CHECK(l.take(300) == 512 && l.end == 812);
    CHECK(l.take(256) == 1024 && l.end == 1280);
    CHECK(l.take(4) == 1280);
    const stage::Dump d(3, 24);
    CHECK(d.recs == 0 && d.addrs == 256 && d.count == 512 && d.l.end == 516);
}

// A staging pair and the calls made through it.
struct Rig {
    std::vector<uint8_t> dev = std::vector<uint8_t>(1 << 16), host = std::vector<uint8_t>(1 << 16);
    std::vector<size_t> asked;   // bytes asked of bufs, per chunk
    std::vector<uint64_t> ks;    // items per launch
    bool refuse = false;
    long syncs0 = S.syncs, h2d0 = S.by_kind[cudaMemcpyHostToDevice], d2h0 = S.by_kind[cudaMemcpyDeviceToHost];
    long syncs() const { return S.syncs - syncs0; }
    long h2d() const { return S.by_kind[cudaMemcpyHostToDevice] - h2d0; }
    long d2h() const { return S.by_kind[cudaMemcpyDeviceToHost] - d2h0; }
    auto bufs() {
        return [this](size_t bytes, uint8_t **d, uint8_t **h) {
            asked.push_back(bytes);
            *d = dev.data(), *h = host.data();
            return !refuse;
        };
    }
    // the "kernel": x = a + b, y = a * 3 for each item; checks where the columns are
    auto launch() {
        return [this](uint8_t *const *d, uint64_t k) {
            ks.push_back(k);
            const size_t off[4] = {size_t(d[0] - dev.data()), size_t(d[1] - dev.data()), size_t(d[2] - dev.data()), size_t(d[3] - dev.data())};
            CHECK(off[0] == 0);
            for (int i = 1; i < 4; i++) CHECK(off[i] % 256 == 0 && off[i] > off[i - 1]);
            CHECK(off[1] >= k * 4 && off[2] >= off[1] + k * 2 && off[3] >= off[2] + k * 4); // inputs, then outputs
            for (uint64_t i = 0; i < k; i++) {
                const uint32_t a = ((const uint32_t *)d[0])[i];
                ((uint32_t *)d[2])[i] = a + ((const uint16_t *)d[1])[i];
                ((uint64_t *)d[3])[i] = 3ull * a;
            }
            return cudaSuccess;
        };
    }
};

static void chunks() {
    const uint64_t sizes[] = {0, 1, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK + 1};
    for (uint64_t n : sizes) {
        std::vector<uint32_t> a(n), x(n, 7);
        std::vector<uint16_t> b(n);
        std::vector<uint64_t> y(n, 7);
        for (uint64_t i = 0; i < n; i++) a[i] = 1000 + (uint32_t)i, b[i] = (uint16_t)(5 * i);
        Rig r;
        const cudaError_t e = stage::round_trip(n, CHUNK, {{a.data(), 4}, {b.data(), 2}}, {{x.data(), 4}, {y.data(), 8}}, nullptr, r.bufs(), r.launch());
        CHECK(e == cudaSuccess);
        const uint64_t nchunks = (n + CHUNK - 1) / CHUNK;
        CHECK(r.ks.size() == nchunks && r.asked.size() == nchunks);
        for (uint64_t c = 0; c < r.ks.size(); c++) {
            const uint64_t k = c + 1 < nchunks ? CHUNK : n - c * CHUNK;
            CHECK(r.ks[c] == k);
            CHECK(r.asked[c] == 768 + k * 8); // a at 0, b at 256, x at 512, y at 768 while k <= 64
        }
        CHECK(r.h2d() == (long)nchunks && r.d2h() == (long)nchunks && r.syncs() == (long)nchunks);
        bool ok = true;
        for (uint64_t i = 0; i < n; i++) ok &= x[i] == a[i] + b[i] && y[i] == 3ull * a[i];
        CHECK(ok);
    }
}

// no output goes back to the host and nobody reads them: no copy back, one synchronisation per chunk all the same
static void no_copy_back() {
    const uint64_t n = 2 * CHUNK + 1;
    std::vector<uint32_t> a(n, 1);
    std::vector<uint16_t> b(n, 2);
    Rig r;
    CHECK(stage::round_trip(n, CHUNK, {{a.data(), 4}, {b.data(), 2}}, {{nullptr, 4}, {nullptr, 8}}, nullptr, r.bufs(), r.launch()) == cudaSuccess);
    CHECK(r.h2d() == 3 && r.d2h() == 0 && r.syncs() == 3);
}

// outputs read in the pinned buffer by the chunk callback, none of them copied out by the round trip
static void chunk_done() {
    const uint64_t n = CHUNK + 3;
    std::vector<uint32_t> a(n), x(n, 0);
    std::vector<uint16_t> b(n, 1);
    for (uint64_t i = 0; i < n; i++) a[i] = (uint32_t)i;
    Rig r;
    uint64_t seen = 0;
    auto done = [&](const uint8_t *const *h, uint64_t at, uint64_t k) {
        CHECK(at == seen);
        for (uint64_t i = 0; i < k; i++)
            if (((const uint64_t *)h[3])[i] % 2 == 0) x[at + i] = ((const uint32_t *)h[2])[i];
        seen += k;
    };
    CHECK(stage::round_trip(n, CHUNK, {{a.data(), 4}, {b.data(), 2}}, {{nullptr, 4}, {nullptr, 8}}, nullptr, r.bufs(), r.launch(), done) == cudaSuccess);
    CHECK(seen == n && r.d2h() == 2 && r.syncs() == 2);
    bool ok = true;
    for (uint64_t i = 0; i < n; i++) ok &= x[i] == (i % 2 == 0 ? a[i] + 1 : 0);
    CHECK(ok);
}

// A failure in the second of three chunks: the first chunk's outputs are delivered, the second's and third's are not,
// nothing runs after it, and its error is returned.
static void failures_stop() {
    const uint64_t n = 2 * CHUNK + 1;
    std::vector<uint32_t> a(n, 4);
    std::vector<uint16_t> b(n, 1);
    auto run = [&](Rig &r, std::vector<uint32_t> &x) {
        std::vector<uint64_t> y(n, 0);
        return stage::round_trip(n, CHUNK, {{a.data(), 4}, {b.data(), 2}}, {{x.data(), 4}, {y.data(), 8}}, nullptr, r.bufs(), r.launch());
    };
    auto first_only = [&](const std::vector<uint32_t> &x) {
        bool ok = true;
        for (uint64_t i = 0; i < n; i++) ok &= x[i] == (i < CHUNK ? 5u : 0u);
        return ok;
    };
    for (long which : {2, 3}) { // the second chunk's copy in (2) or back (3)
        Rig r;
        std::vector<uint32_t> x(n, 0);
        S.fail_copy_at = S.copies + which;
        CHECK(run(r, x) == cudaErrorLaunchFailure);
        CHECK(first_only(x));
        CHECK(r.ks.size() == (which == 2 ? 1u : 2u) && r.syncs() == 1);
        cudaGetLastError();
    }
    {
        Rig r;
        std::vector<uint32_t> x(n, 0);
        auto launch = r.launch();
        auto failing = [&](uint8_t *const *d, uint64_t k) {
            launch(d, k);
            if (r.ks.size() == 2) S.fail_sync = true; // the second chunk's kernel faults
            return cudaSuccess;
        };
        CHECK(stage::round_trip(n, CHUNK, {{a.data(), 4}, {b.data(), 2}}, {{x.data(), 4}, {nullptr, 8}}, nullptr, r.bufs(), failing) ==
              cudaErrorLaunchFailure);
        CHECK(first_only(x) && r.ks.size() == 2 && r.syncs() == 2 && r.d2h() == 2);
        cudaGetLastError();
    }
    {
        Rig r;
        std::vector<uint32_t> x(n, 0);
        auto launch = r.launch();
        auto refusing = [&](uint8_t *const *d, uint64_t k) {
            launch(d, k);
            return r.ks.size() == 2 ? cudaErrorLaunchFailure : cudaSuccess; // the second chunk's launch is refused
        };
        CHECK(stage::round_trip(n, CHUNK, {{a.data(), 4}, {b.data(), 2}}, {{x.data(), 4}, {nullptr, 8}}, nullptr, r.bufs(), refusing) ==
              cudaErrorLaunchFailure);
        CHECK(first_only(x) && r.ks.size() == 2 && r.d2h() == 1 && r.syncs() == 1);
    }
    {
        Rig r;
        r.refuse = true;
        std::vector<uint32_t> x(n, 0);
        CHECK(run(r, x) == cudaErrorMemoryAllocation && r.ks.empty() && r.h2d() == 0 && r.asked.size() == 1);
    }
}

static void counted_dump() {
    std::vector<uint8_t> buf(2048, 0xEE);
    for (uint32_t found : {0u, 2u, 3u, 5u}) {
        const uint64_t cap = 3;
        std::vector<uint64_t> recs(cap + 1, 0);
        std::vector<uint32_t> addrs(cap + 1, 0);
        uint32_t count = 99;
        auto launch = [&](uint8_t *r, uint32_t *a, uint32_t *cnt) {
            CHECK(*cnt == 0); // zeroed before the launch
            for (uint32_t i = 0; i < found && i < cap; i++) ((uint64_t *)r)[i] = 100 + i, a[i] = 10 + i;
            *cnt = found;
            return cudaSuccess;
        };
        const long copies = S.copies;
        CHECK(stage::counted_dump(buf.data(), cap, 8, recs.data(), addrs.data(), &count, nullptr, launch) == cudaSuccess);
        CHECK(count == found);
        const uint32_t got = found < cap ? found : cap;
        CHECK(S.copies - copies == (got ? 3 : 1));
        bool ok = true;
        for (uint32_t i = 0; i <= cap; i++) ok &= recs[i] == (i < got ? 100 + i : 0) && addrs[i] == (i < got ? 10 + i : 0);
        CHECK(ok);
    }
}

int main() {
    layout();
    chunks();
    no_copy_back();
    chunk_done();
    failures_stop();
    counted_dump();
    CHECK(S.live.empty());
    if (failures) return 1;
    printf("stage host test ok\n");
    return 0;
}
