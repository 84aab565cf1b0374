// Host-device staging of the control-plane calls (ctx.cu).  It needs nothing but the runtime API, so that a host test
// can build it against a fake runtime (tests/host/test_stage_host.cpp).
#pragma once
#include <cuda_runtime_api.h>
#include <stdint.h>
#include <string.h>

#include <initializer_list>
#include <type_traits>
#include <vector>

namespace stage {

// Regions of one buffer laid end to end, each starting at a 256-byte boundary, in the order they are taken.
struct Layout {
    size_t end = 0; // the end of the last region taken
    size_t take(size_t bytes) {
        const size_t at = (end + 255) & ~(size_t)255;
        end = at + bytes;
        return at;
    }
};

// A column of items in host memory, item i at host + i * size.  A null input is not staged; a null output is not
// copied out (chunk_done may read it in the pinned buffer).
struct In { const void *host; size_t size; };
struct Out { void *host; size_t size; };

// n items in chunks of at most `chunk` through a device buffer and its pinned twin, bufs(bytes, &dev, &host) -> bool
// (false: cudaErrorMemoryAllocation, the callback reports why).  Each chunk lays its inputs out before its outputs,
// stages the inputs, copies them to the device in one copy, runs launch(dev_cols, k) -> cudaError_t, copies the
// outputs back in one copy (none when no output has a host and there is no chunk_done), synchronises `st` once, copies
// the outputs out and runs chunk_done(pinned_cols, done, k).  The first error ends the loop and is returned.
template <class Bufs, class Launch, class Done = std::nullptr_t>
cudaError_t round_trip(uint64_t n, uint64_t chunk, std::initializer_list<In> in, std::initializer_list<Out> out, cudaStream_t st,
                       Bufs bufs, Launch launch, Done chunk_done = nullptr) {
    constexpr bool reads = !std::is_null_pointer<Done>::value;
    bool back = reads;
    for (const Out &o : out) back = back || o.host;
    std::vector<size_t> off(in.size() + out.size());
    std::vector<uint8_t *> d(off.size()), h(off.size());
    for (uint64_t done = 0; done < n; done += chunk) {
        const uint64_t k = n - done < chunk ? n - done : chunk;
        Layout l;
        size_t i = 0;
        for (const In &c : in) off[i++] = l.take(k * c.size);
        const size_t in_end = l.end, out0 = l.take(0);
        for (const Out &c : out) off[i++] = l.take(k * c.size);
        uint8_t *dev, *host;
        if (!bufs(l.end, &dev, &host)) return cudaErrorMemoryAllocation;
        for (i = 0; i < off.size(); i++) d[i] = dev + off[i], h[i] = host + off[i];
        i = 0;
        for (const In &c : in) {
            if (c.host) memcpy(h[i], (const uint8_t *)c.host + done * c.size, k * c.size);
            i++;
        }
        cudaError_t e = cudaMemcpyAsync(dev, host, in_end, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = launch(d.data(), k);
        if (e == cudaSuccess && back) e = cudaMemcpyAsync(host + out0, dev + out0, l.end - out0, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return e;
        for (const Out &c : out) {
            if (c.host) memcpy((uint8_t *)c.host + done * c.size, h[i], k * c.size);
            i++;
        }
        if constexpr (reads) chunk_done((const uint8_t *const *)h.data(), done, k);
    }
    return cudaSuccess;
}

// A counted dump's device buffer for `cap` records of `rec` bytes: the records, then their addresses, then the count.
struct Dump {
    Layout l;
    size_t recs, addrs, count;
    Dump(uint64_t cap, size_t rec) : recs(l.take(cap * rec)), addrs(l.take(cap * 4)), count(l.take(4)) {}
};

// launch(recs, addrs, count) -> cudaError_t writes a dump into `buf` (Dump(cap, rec).l.end bytes of device memory), its
// count from zero.  *count is the count it reported, which may exceed cap; min(*count, cap) records and addresses are
// copied out.
template <class Launch>
cudaError_t counted_dump(uint8_t *buf, uint64_t cap, size_t rec, void *recs_out, uint32_t *addrs_out, uint32_t *count,
                         cudaStream_t st, Launch launch) {
    const Dump d(cap, rec);
    uint32_t *cnt = (uint32_t *)(buf + d.count);
    *count = 0;
    cudaError_t e = cudaMemsetAsync(cnt, 0, 4, st);
    if (e == cudaSuccess) e = launch(buf + d.recs, (uint32_t *)(buf + d.addrs), cnt);
    if (e == cudaSuccess) e = cudaMemcpyAsync(count, cnt, 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    const uint64_t got = *count < cap ? *count : cap;
    if (e == cudaSuccess && got) e = cudaMemcpy(recs_out, buf + d.recs, got * rec, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && got) e = cudaMemcpy(addrs_out, buf + d.addrs, got * 4, cudaMemcpyDeviceToHost);
    return e;
}

} // namespace stage
