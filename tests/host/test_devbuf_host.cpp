// The context's buffer owners (bng_b200/csrc/devbuf.hpp) against a fake runtime (fake_cuda/cuda_runtime_api.h): what a
// failed growth leaves behind, all-or-none growth of a set, and that every allocation is freed once, by the right call.
#include <cstdio>

#include "../../bng_b200/csrc/devbuf.hpp"

static int failures = 0;
#define CHECK(c)                                                             \
    do {                                                                     \
        if (!(c)) {                                                          \
            fprintf(stderr, "%s:%d: CHECK failed: %s\n", __FILE__, __LINE__, #c); \
            failures++;                                                      \
        }                                                                    \
    } while (0)

static fake::State &S = fake::st();

static void fail_next_alloc(long k = 0) { S.fail_at = S.allocs + k; }

static void discarding_growth() {
    DevBuf<unsigned> b;
    CHECK(b.grow(64) && b.get() && b.size() == 64);
    unsigned *p = b;
    CHECK(b.grow(64) && b.get() == p); // holds as many already: nothing happens
    CHECK(b.grow(16) && b.get() == p && b.size() == 64);
    CHECK(b.grow(0) && b.get() == p);
    fail_next_alloc();
    CHECK(!b.grow(128));
    CHECK(b.get() == nullptr && b.size() == 0 && !b);
    CHECK(S.last == cudaSuccess);
    CHECK(S.live.empty());
    CHECK(b.grow(128) && b.size() == 128); // the next growth starts from empty
}

static void replacing_growth() {
    DevBuf<unsigned char> b;
    CHECK(b.grow(64));
    for (int i = 0; i < 64; i++) b[i] = (unsigned char)i;
    unsigned char *p = b;
    fail_next_alloc();
    CHECK(b.grow_keep(128, 32, nullptr) == cudaErrorMemoryAllocation);
    CHECK(b.get() == p && b.size() == 64);
    bool same = true;
    for (int i = 0; i < 64; i++) same &= b[i] == i;
    CHECK(same);
    CHECK(S.last == cudaSuccess);
    CHECK(S.live.size() == 1);
    // a failed synchronisation (an earlier launch's error) is the caller's to report: not cleared, not an allocation
    S.fail_sync = true;
    CHECK(b.grow_keep(128, 32, nullptr) == cudaErrorLaunchFailure);
    CHECK(b.get() == p && b.size() == 64 && S.live.size() == 1);
    CHECK(cudaGetLastError() == cudaErrorLaunchFailure);
    const long syncs = S.syncs;
    CHECK(b.grow_keep(128, 32, nullptr) == cudaSuccess && b.size() == 128 && b.get() != p);
    CHECK(S.syncs == syncs + 1); // the old allocation is freed only after the stream is done with it
    same = true;
    for (int i = 0; i < 32; i++) same &= b[i] == i;
    CHECK(same);
    CHECK(S.live.size() == 1 && S.live.count(b.get()));
}

static void group_growth() {
    DevBuf<unsigned> a, c;
    PinnedBuf<unsigned char> h;
    CHECK(a.grow(16));
    fail_next_alloc(2); // the third allocation of the set, by the third member
    CHECK(!devbuf::grow_all({{&a, 64}, {&h, 64}, {&c, 64}}));
    CHECK(!a && !h && !c && a.size() == 0 && h.size() == 0 && c.size() == 0);
    CHECK(S.last == cudaSuccess);
    CHECK(S.live.empty());
    CHECK(devbuf::grow_all({{&a, 64}, {&h, 64}, {&c, 0}}));
    CHECK(a.size() == 64 && h.size() == 64 && !c);
    CHECK(S.live.size() == 2 && S.live[h.get()] == fake::HOST && S.live[a.get()] == fake::DEV);
}

static void frees_once() {
    {
        DevBuf<unsigned> a, b;
        PinnedBuf<unsigned long long> h;
        CHECK(a.grow(8) && b.grow(8) && h.grow(8));
        DevBuf<unsigned> m(static_cast<DevBuf<unsigned> &&>(a)); // moved from: a is empty
        CHECK(!a && m);
        b = static_cast<DevBuf<unsigned> &&>(m); // b's old allocation is freed, m's moves over
        CHECK(!m && b && S.live.size() == 2);
        void *raw = nullptr;
        CHECK(cudaMalloc(&raw, 8) == cudaSuccess);
        DevBuf<unsigned> adopted((unsigned *)raw, 8);
        DevBuf<unsigned> released;
        CHECK(released.grow(8));
        unsigned *kept = released.release();
        CHECK(!released && S.live.count(kept));
        cudaFree(kept);
        CHECK(S.live.size() == 3);
    }
    CHECK(S.live.empty());
    CHECK(S.bad_frees == 0);
}

int main() {
    discarding_growth();
    replacing_growth();
    group_growth();
    frees_once();
    CHECK(S.live.empty() && S.bad_frees == 0);
    if (failures) {
        fprintf(stderr, "%d check(s) failed\n", failures);
        return 1;
    }
    printf("devbuf host tests ok\n");
    return 0;
}
