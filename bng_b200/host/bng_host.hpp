// bng_host.hpp — host side of the dataplane boundary, in C++ (the Go toolchain
// the reference's host code is written in is not available in this image).
//
// Mirrors, name for name, the Go types that own the reference's eBPF objects:
//   bng::ebpf::Loader       pkg/ebpf/loader.go:74-706        (DHCP fast path maps)
//   bng::antispoof::Manager pkg/antispoof/manager.go:16-399
//   bng::qos::Manager       pkg/qos/manager.go:16-327
//   bng::nat::Manager       pkg/nat/manager.go:17-845        (incl. the host-side port-block allocator)
// with `*ebpf.Collection / *ebpf.Map` replaced by a bng_ctx handle and map ids
// of the C ABI in include/bng_b200.h.  Same argument meaning, same bookkeeping,
// same error strings ("<name> map not loaded" before Load/Start, tested by the
// reference in pkg/ebpf/loader_test.go:383-446).  Go's (value, error) returns
// become Result<T>; a Go `error` becomes bng::Error (empty message = nil).
//
// Byte order: like the Go code, addresses cross this API as uint32 values
// obtained with BigEndian.Uint32 and are written to the maps in host (little-
// endian) order — i.e. byte-reversed with respect to the wire, which the eBPF
// programs (and therefore the kernels) compare against verbatim.  That is the
// reference's behaviour (SURVEY.md §7.3-3); set Backend::wire_order_keys to
// store addresses in wire order instead, so that control-plane entries match
// real frames.
#pragma once

#include <chrono>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <string>
#include <vector>

#include "../../include/bng_b200.h"

namespace bng {

struct Error {
    std::string msg;
    Error() = default;
    explicit Error(std::string m) : msg(std::move(m)) {}
    explicit operator bool() const { return !msg.empty(); } // true = there IS an error (Go: err != nil)
    const std::string &what() const { return msg; }
};
inline Error Nil() { return Error(); }

template <class T>
struct Result {
    std::optional<T> value;
    Error err;
    bool ok() const { return !err; }
    T *operator->() { return &*value; }
    T &operator*() { return *value; }
};

using IP = std::vector<uint8_t>;  // net.IP: 4 or 16 bytes
using MAC = std::vector<uint8_t>; // net.HardwareAddr

inline IP IPv4(uint8_t a, uint8_t b, uint8_t c, uint8_t d) { return IP{a, b, c, d}; }
inline const uint8_t *To4(const IP &ip) { // net.IP.To4()
    if (ip.size() == 4) return ip.data();
    if (ip.size() == 16) {
        static const uint8_t pfx[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0xff, 0xff};
        if (!memcmp(ip.data(), pfx, 12)) return ip.data() + 12;
    }
    return nullptr;
}

// One dataplane context shared by the managers of a process (the reference loads
// four collections whose map names are disjoint; one context holds all of them).
struct Backend {
    bng_ctx *ctx = nullptr;
    bool wire_order_keys = false;
    std::string open_error;
    ~Backend() {
        if (ctx) bng_close(ctx);
    }
    static std::shared_ptr<Backend> Open(const bng_open_opts *opts = nullptr) {
        auto b = std::make_shared<Backend>();
        b->ctx = bng_open(opts);
        if (!b->ctx) b->open_error = bng_last_error(nullptr);
        return b;
    }
    int Map(const char *name) const { return ctx ? bng_map_id(ctx, name) : -1; }
    uint32_t AddrKey(uint32_t be_numeric) const { // what lands in the map for an address given as BigEndian.Uint32
        return wire_order_keys ? __builtin_bswap32(be_numeric) : be_numeric;
    }
};

inline Error MapErr(const char *what, int rc) {
    if (rc == 0) return Nil();
    return Error(std::string(what) + ": errno " + std::to_string(-rc));
}

// ===========================================================================
// RADIUS accounting counters (reference pkg/radius/accounting.go:128-137: SessionCounters and the CounterFetcher
// callback that SetCounterFetcher installs).  Acct-Input-* is traffic FROM the user: the upstream pass pair of the
// subscriber's bng_acct record; Acct-Output-* the downstream pass pair.
namespace radius {

struct SessionCounters {
    uint64_t InputOctets = 0, OutputOctets = 0, InputPackets = 0, OutputPackets = 0;
};

inline SessionCounters CountersOf(const bng_acct &a) {
    SessionCounters s;
    s.InputOctets = a.up_bytes;
    s.InputPackets = a.up_packets;
    s.OutputOctets = a.down_bytes;
    s.OutputPackets = a.down_packets;
    return s;
}

// func(sessionID string) (*SessionCounters, error)
using CounterFetcher = std::function<Result<SessionCounters>(const std::string &session_id)>;
// session id -> the subscriber's IPv4 address as the qos_ingress key holds it (the accounting manager knows the
// Framed-IP-Address of every session it started)
using SessionAddr = std::function<std::optional<uint32_t>(const std::string &session_id)>;
// reads one subscriber's record: 0, -ENOENT or a negative errno
using AcctReader = std::function<int(uint32_t addr_key, bng_acct *out)>;

inline CounterFetcher MakeCounterFetcher(SessionAddr addr_of, AcctReader read) {
    return [addr_of = std::move(addr_of), read = std::move(read)](const std::string &id) {
        Result<SessionCounters> r;
        auto a = addr_of(id);
        if (!a) {
            r.err = Error("session " + id + ": no address");
            return r;
        }
        bng_acct rec{};
        if (Error e = MapErr("bng_acct_read", read(*a, &rec))) {
            r.err = e;
            return r;
        }
        r.value = CountersOf(rec);
        return r;
    };
}

// the reader of one context
inline AcctReader ContextReader(std::shared_ptr<Backend> b) {
    return [b = std::move(b)](uint32_t addr, bng_acct *out) {
        int32_t res = 0;
        int rc = bng_acct_read(b->ctx, &addr, 1, out, &res);
        return rc ? rc : res;
    };
}

} // namespace radius

// ===========================================================================
// Lawful intercept, content of communication (reference pkg/intercept/manager.go:337: Manager.RecordCC(warrant,
// session, direction, srcIP, dstIP, srcPort, dstPort, protocol, payload)).  StartInterceptSession sets the session's
// IPv4 address as a target (bng_li_target_set), StopInterceptSession deletes it; PumpCC drains the records and hands
// each one, parsed into RecordCC's arguments, to the caller.
namespace intercept {

enum class Direction : uint8_t { Uplink = BNG_LI_UPLINK, Downlink = BNG_LI_DOWNLINK };

struct CC {
    bng_li_record rec;                // the record's header: target, frame, batch, verdict, timestamp
    Direction direction = Direction::Uplink;
    IP src, dst;                      // 4 bytes each, wire order; 0.0.0.0 when the capture is too short for it
    uint16_t src_port = 0, dst_port = 0; // host order
    uint8_t protocol = 0;
    std::vector<uint8_t> payload;     // the IP packet as captured: bytes 14 .. cap_len of the frame
};

// The fields RecordCC takes, from one record (header + cap_len captured bytes).  Ports: TCP / UDP source and
// destination port at 14 + 4 * ihl; ICMP echo request / reply: the echo id, which the NAT translates in place of a port,
// as the subscriber-side port (src_port uplink, dst_port downlink); 0 for any other protocol or when the capture ends
// before them.  Returns false when the capture does not hold the IPv4 header's first 20 bytes' addresses.
inline bool ParseCC(const uint8_t *record, CC *out) {
    memcpy(&out->rec, record, sizeof(bng_li_record));
    const uint8_t *f = record + sizeof(bng_li_record);
    const uint32_t n = out->rec.cap_len;
    out->direction = out->rec.dir == BNG_LI_DOWNLINK ? Direction::Downlink : Direction::Uplink;
    out->src = n >= 30 ? IP(f + 26, f + 30) : IPv4(0, 0, 0, 0);
    out->dst = n >= 34 ? IP(f + 30, f + 34) : IPv4(0, 0, 0, 0);
    out->protocol = n >= 24 ? f[23] : 0;
    out->src_port = out->dst_port = 0;
    out->payload.assign(f + (n > 14 ? 14 : n), f + n);
    if (n < 34) return false;
    const uint32_t l4 = 14 + 4u * (f[14] & 0x0f);
    auto be16 = [&](uint32_t off) { return (uint16_t)(f[off] << 8 | f[off + 1]); };
    if ((out->protocol == 6 || out->protocol == 17) && n >= l4 + 4) {
        out->src_port = be16(l4);
        out->dst_port = be16(l4 + 2);
    } else if (out->protocol == 1 && n >= l4 + 6 && (f[l4] == 0 || f[l4] == 8)) {
        (out->direction == Direction::Uplink ? out->src_port : out->dst_port) = be16(l4 + 4);
    }
    return true;
}

// The caller's warrant / session of a target id, or none: the record is skipped (an IRI-only warrant, a session that
// ended while its records were queued), as RecordCC skips them.
template <class W>
using Resolver = std::function<std::optional<W>(uint32_t target_id)>;
template <class W>
using Sink = std::function<void(const W &warrant, const CC &cc)>;

// records laid out as bng_li_drain() returns them; returns the number handed to the sink
template <class W>
inline uint64_t PumpRecords(const uint8_t *recs, uint64_t n, uint32_t rec_size, const Resolver<W> &resolve, const Sink<W> &sink) {
    uint64_t done = 0;
    CC cc;
    for (uint64_t i = 0; i < n; i++) {
        const uint8_t *r = recs + i * rec_size;
        uint32_t id;
        memcpy(&id, r + offsetof(bng_li_record, target_id), 4);
        std::optional<W> w = resolve(id);
        if (!w) continue;
        ParseCC(r, &cc);
        sink(*w, cc);
        done++;
    }
    return done;
}

// Drains the context until it is empty, `batch` records per call.  Returns the records handed to the sink, or a
// negative errno.
template <class W>
inline int64_t PumpCC(bng_ctx *ctx, const Resolver<W> &resolve, const Sink<W> &sink, uint64_t batch = 4096) {
    const uint32_t rs = bng_li_record_size(ctx);
    if (!rs) return 0;
    std::vector<uint8_t> buf((size_t)batch * rs);
    int64_t total = 0;
    for (;;) {
        uint64_t n = 0;
        int rc = bng_li_drain(ctx, buf.data(), batch, &n);
        if (rc) return rc;
        total += (int64_t)PumpRecords<W>(buf.data(), n, rs, resolve, sink);
        if (n < batch) return total;
    }
}

} // namespace intercept

// ===========================================================================
namespace ebpf {

#pragma pack(push, 1)
struct PoolAssignment { // pkg/ebpf/loader.go:21-29, bpf/maps.h:89-97 (25 bytes)
    uint32_t PoolID = 0;
    uint32_t AllocatedIP = 0;
    uint32_t VlanID = 0;
    uint8_t ClientClass = 0;
    uint64_t LeaseExpiry = 0;
    uint8_t Flags = 0;
    uint8_t _pad[3] = {0, 0, 0};
};
struct VLANKey { // :34-37
    uint16_t STag = 0, CTag = 0;
};
struct IPPool { // :40-49 (28 bytes)
    uint32_t Network = 0;
    uint8_t PrefixLen = 0;
    uint8_t _pad1[3] = {0, 0, 0};
    uint32_t Gateway = 0, DNSPrimary = 0, DNSSecondary = 0, LeaseTime = 0, _pad2 = 0;
};
struct DHCPStats { // :52-63 (80 bytes)
    uint64_t TotalRequests = 0, FastpathHits = 0, FastpathMisses = 0, Errors = 0, CacheExpired = 0, Option82Present = 0,
             Option82Absent = 0, BroadcastReplies = 0, UnicastReplies = 0, VLANPackets = 0;
};
struct ServerConfig { // :66-71 (16 bytes)
    uint8_t ServerMAC[6] = {0, 0, 0, 0, 0, 0};
    uint8_t _pad[2] = {0, 0};
    uint32_t ServerIP = 0, InterfaceIndex = 0;
};
#pragma pack(pop)
static_assert(sizeof(PoolAssignment) == 25 && sizeof(VLANKey) == 4 && sizeof(IPPool) == 28, "ABI");
static_assert(sizeof(DHCPStats) == 80 && sizeof(ServerConfig) == 16, "ABI");

constexpr int CircuitIDKeyLen = 32; // :616
struct CircuitIDKey {
    uint8_t b[CircuitIDKeyLen] = {0};
};

// --- helpers, :546-553, :620-624, :666-706 ---
inline uint64_t HashCircuitID(const std::vector<uint8_t> &id) { // FNV-1a 64
    uint64_t h = 0xcbf29ce484222325ull;
    for (uint8_t c : id) {
        h ^= c;
        h *= 0x100000001b3ull;
    }
    return h;
}
inline CircuitIDKey MakeCircuitIDKey(const std::vector<uint8_t> &id) {
    CircuitIDKey k;
    memcpy(k.b, id.data(), id.size() < (size_t)CircuitIDKeyLen ? id.size() : (size_t)CircuitIDKeyLen);
    return k;
}
inline uint32_t IPToUint32(const IP &ip) {
    const uint8_t *p = To4(ip);
    if (!p) return 0;
    return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}
inline IP Uint32ToIP(uint32_t n) { return IP{(uint8_t)(n >> 24), (uint8_t)(n >> 16), (uint8_t)(n >> 8), (uint8_t)n}; }
inline uint64_t MACToUint64(const MAC &mac) {
    if (mac.size() < 6) return 0;
    uint64_t r = 0;
    for (int i = 0; i < 6; i++) r = (r << 8) | mac[i];
    return r;
}
inline MAC Uint64ToMAC(uint64_t n) {
    MAC m(6);
    for (int i = 5; i >= 0; i--) {
        m[i] = (uint8_t)(n & 0xff);
        n >>= 8;
    }
    return m;
}
inline uint64_t LeaseExpiryFromDuration(std::chrono::seconds d) {
    return (uint64_t)std::chrono::duration_cast<std::chrono::seconds>((std::chrono::system_clock::now() + d).time_since_epoch())
        .count();
}

class Loader {
  public:
    // NewLoader, :110-127.  `bpfPath` is kept for interface compatibility; it selects nothing here.
    static Result<std::shared_ptr<Loader>> NewLoader(const std::string &iface, std::shared_ptr<Backend> backend = nullptr,
                                                    const std::string &bpfPath = "bpf/dhcp_fastpath.bpf.o") {
        Result<std::shared_ptr<Loader>> r;
        if (iface.empty()) {
            r.err = Error("interface name is required");
            return r;
        }
        auto l = std::shared_ptr<Loader>(new Loader());
        l->iface_ = iface;
        l->bpfPath_ = bpfPath;
        l->be_ = std::move(backend);
        r.value = l;
        return r;
    }
    // Load, :176-323: opens the dataplane context (unless one was handed in), fetches the maps by name,
    // zeroes stats_map.  "Attaching the XDP program" has no equivalent: frames reach the program through
    // bng_prog_run.
    Error Load() {
        if (!be_) be_ = Backend::Open();
        if (!be_->ctx) return Error("failed to load eBPF spec: " + be_->open_error);
        subscriberPools_ = be_->Map("subscriber_pools");
        if (subscriberPools_ < 0) return Error("subscriber_pools map not found");
        vlanSubscriberPools_ = be_->Map("vlan_subscriber_pools");
        ipPools_ = be_->Map("ip_pools");
        if (ipPools_ < 0) return Error("ip_pools map not found");
        statsMap_ = be_->Map("stats_map");
        serverConfigMap_ = be_->Map("server_config");
        circuitIDMap_ = be_->Map("circuit_id_map");
        circuitIDSubscribers_ = be_->Map("circuit_id_subscribers");
        loaded_ = true;
        return ResetStats();
    }
    Error Close() { // idempotent, loader_test.go:989-1003
        loaded_ = false;
        subscriberPools_ = vlanSubscriberPools_ = ipPools_ = statsMap_ = serverConfigMap_ = circuitIDMap_ = circuitIDSubscribers_ = -1;
        be_.reset();
        return Nil();
    }
    std::shared_ptr<Backend> backend() const { return be_; }

    Error AddSubscriber(uint64_t mac, const PoolAssignment &a) {
        if (subscriberPools_ < 0) return Error("subscriber_pools map not loaded");
        return MapErr("update", bng_map_update(be_->ctx, subscriberPools_, &mac, &a, BNG_ANY));
    }
    Error RemoveSubscriber(uint64_t mac) {
        if (subscriberPools_ < 0) return Error("subscriber_pools map not loaded");
        return MapErr("delete", bng_map_delete(be_->ctx, subscriberPools_, &mac));
    }
    Result<PoolAssignment> GetSubscriber(uint64_t mac) { return lookup<PoolAssignment>(subscriberPools_, "subscriber_pools map not loaded", &mac); }

    Error AddVLANSubscriber(uint16_t sTag, uint16_t cTag, const PoolAssignment &a) {
        if (vlanSubscriberPools_ < 0) return Error("vlan_subscriber_pools map not loaded");
        VLANKey k{sTag, cTag};
        return MapErr("update", bng_map_update(be_->ctx, vlanSubscriberPools_, &k, &a, BNG_ANY));
    }
    Error RemoveVLANSubscriber(uint16_t sTag, uint16_t cTag) {
        if (vlanSubscriberPools_ < 0) return Error("vlan_subscriber_pools map not loaded");
        VLANKey k{sTag, cTag};
        return MapErr("delete", bng_map_delete(be_->ctx, vlanSubscriberPools_, &k));
    }
    Result<PoolAssignment> GetVLANSubscriber(uint16_t sTag, uint16_t cTag) {
        VLANKey k{sTag, cTag};
        return lookup<PoolAssignment>(vlanSubscriberPools_, "vlan_subscriber_pools map not loaded", &k);
    }
    bool HasVLANSupport() const { return vlanSubscriberPools_ >= 0; }

    Error AddPool(uint32_t poolID, const IPPool &p) {
        if (ipPools_ < 0) return Error("ip_pools map not loaded");
        return MapErr("update", bng_map_update(be_->ctx, ipPools_, &poolID, &p, BNG_ANY));
    }
    Error RemovePool(uint32_t poolID) {
        if (ipPools_ < 0) return Error("ip_pools map not loaded");
        return MapErr("delete", bng_map_delete(be_->ctx, ipPools_, &poolID));
    }
    Result<IPPool> GetPool(uint32_t poolID) { return lookup<IPPool>(ipPools_, "ip_pools map not loaded", &poolID); }

    Result<DHCPStats> GetStats() {
        uint32_t key = 0;
        return lookup<DHCPStats>(statsMap_, "stats_map not loaded", &key);
    }
    Error ResetStats() {
        if (statsMap_ < 0) return Error("stats_map not loaded");
        uint32_t key = 0;
        DHCPStats z;
        return MapErr("update", bng_map_update(be_->ctx, statsMap_, &key, &z, BNG_ANY));
    }
    Error SetServerConfig(const MAC &serverMAC, const IP &serverIP, int ifIndex) { // :485-499
        if (serverConfigMap_ < 0) return Error("server_config map not loaded");
        ServerConfig c;
        if (serverMAC.size() >= 6) memcpy(c.ServerMAC, serverMAC.data(), 6);
        c.ServerIP = be_->AddrKey(IPToUint32(serverIP));
        c.InterfaceIndex = (uint32_t)ifIndex;
        uint32_t key = 0;
        return MapErr("update", bng_map_update(be_->ctx, serverConfigMap_, &key, &c, BNG_ANY));
    }
    Result<ServerConfig> GetServerConfig() {
        uint32_t key = 0;
        return lookup<ServerConfig>(serverConfigMap_, "server_config map not loaded", &key);
    }

    Error AddCircuitIDMapping(const std::vector<uint8_t> &id, uint64_t mac) {
        if (circuitIDMap_ < 0) return Error("circuit_id_map not loaded");
        uint64_t h = HashCircuitID(id);
        return MapErr("update", bng_map_update(be_->ctx, circuitIDMap_, &h, &mac, BNG_ANY));
    }
    Error RemoveCircuitIDMapping(const std::vector<uint8_t> &id) {
        if (circuitIDMap_ < 0) return Error("circuit_id_map not loaded");
        uint64_t h = HashCircuitID(id);
        return MapErr("delete", bng_map_delete(be_->ctx, circuitIDMap_, &h));
    }
    Result<uint64_t> GetCircuitIDMapping(const std::vector<uint8_t> &id) {
        uint64_t h = HashCircuitID(id);
        return lookup<uint64_t>(circuitIDMap_, "circuit_id_map not loaded", &h);
    }
    Result<bool> CheckCircuitIDCollision(const std::vector<uint8_t> &id, uint64_t newMAC) { // :594-609
        Result<bool> r;
        if (circuitIDMap_ < 0) {
            r.err = Error("circuit_id_map not loaded");
            r.value = false;
            return r;
        }
        auto e = GetCircuitIDMapping(id);
        r.value = e.ok() ? (*e.value != newMAC) : false;
        return r;
    }
    Error AddCircuitIDSubscriber(const std::vector<uint8_t> &id, const PoolAssignment &a) {
        if (circuitIDSubscribers_ < 0) return Error("circuit_id_subscribers map not loaded");
        CircuitIDKey k = MakeCircuitIDKey(id);
        return MapErr("update", bng_map_update(be_->ctx, circuitIDSubscribers_, &k, &a, BNG_ANY));
    }
    Error RemoveCircuitIDSubscriber(const std::vector<uint8_t> &id) {
        if (circuitIDSubscribers_ < 0) return Error("circuit_id_subscribers map not loaded");
        CircuitIDKey k = MakeCircuitIDKey(id);
        return MapErr("delete", bng_map_delete(be_->ctx, circuitIDSubscribers_, &k));
    }
    Result<PoolAssignment> GetCircuitIDSubscriber(const std::vector<uint8_t> &id) {
        CircuitIDKey k = MakeCircuitIDKey(id);
        return lookup<PoolAssignment>(circuitIDSubscribers_, "circuit_id_subscribers map not loaded", &k);
    }
    bool HasCircuitIDSubscriberSupport() const { return circuitIDSubscribers_ >= 0; }

  private:
    Loader() = default;
    template <class T>
    Result<T> lookup(int map, const char *unloaded, const void *key) {
        Result<T> r;
        if (map < 0) {
            r.err = Error(unloaded);
            return r;
        }
        T v{};
        int rc = bng_map_lookup(be_->ctx, map, key, &v);
        if (rc)
            r.err = MapErr("lookup", rc);
        else
            r.value = v;
        return r;
    }
    std::string iface_, bpfPath_;
    std::shared_ptr<Backend> be_;
    bool loaded_ = false;
    int subscriberPools_ = -1, vlanSubscriberPools_ = -1, ipPools_ = -1, statsMap_ = -1, serverConfigMap_ = -1,
        circuitIDMap_ = -1, circuitIDSubscribers_ = -1;
};

} // namespace ebpf

// ===========================================================================
namespace antispoof {

enum Mode : uint8_t { ModeDisabled = 0, ModeStrict = 1, ModeLoose = 2, ModeLogOnly = 3 }; // manager.go:19-30

#pragma pack(push, 1)
struct SubscriberBinding { // :33-40, bpf/antispoof.c:36-43 (24 bytes)
    uint32_t IPv4Addr = 0;
    uint8_t IPv6Addr[16] = {0};
    uint8_t IPv4Valid = 0, IPv6Valid = 0, Mode = 0, _pad = 0;
};
struct Config { // :43-47
    uint8_t DefaultMode = 0, LogViolations = 0, _pad[6] = {0, 0, 0, 0, 0, 0};
};
struct Stats { // :50-57 (48 bytes)
    uint64_t PacketsAllowed = 0, PacketsDropped = 0, PacketsLogged = 0, IPv4Violations = 0, IPv6Violations = 0, UnknownMAC = 0;
};
struct SpoofEvent { // :60-69 (56 bytes)
    uint64_t Timestamp;
    uint8_t SrcMAC[6], Protocol, _pad;
    uint32_t SpoofedIP, AllowedIP;
    uint8_t SpoofedIPv6[16], AllowedIPv6[16];
};
#pragma pack(pop)
static_assert(sizeof(SubscriberBinding) == 24 && sizeof(Config) == 8 && sizeof(Stats) == 48 && sizeof(SpoofEvent) == 56, "ABI");

struct ManagerConfig { // :89-94
    std::string Interface, BPFPath;
    Mode DefaultMode = ModeDisabled;
    bool LogViolations = true;
    std::shared_ptr<Backend> Backend_;
};

class Manager {
  public:
    static Result<std::shared_ptr<Manager>> NewManager(const ManagerConfig &cfg) { // :102-124
        Result<std::shared_ptr<Manager>> r;
        if (cfg.Interface.empty()) {
            r.err = Error("interface required");
            return r;
        }
        auto m = std::shared_ptr<Manager>(new Manager());
        m->cfg_ = cfg;
        m->mode_ = cfg.DefaultMode;
        m->be_ = cfg.Backend_;
        r.value = m;
        return r;
    }
    Error Start() { // :127-186: load, grab maps, write the config entry, attach
        if (!be_) be_ = Backend::Open();
        if (!be_->ctx) return Error("failed to load eBPF spec: " + be_->open_error);
        bindings_ = be_->Map("subscriber_bindings");
        if (bindings_ < 0) return Error("subscriber_bindings map not found");
        config_ = be_->Map("antispoof_config");
        stats_ = be_->Map("antispoof_stats");
        ranges_ = be_->Map("allowed_ranges_v4");
        if (config_ >= 0) {
            Config c;
            c.DefaultMode = (uint8_t)mode_;
            c.LogViolations = cfg_.LogViolations ? 1 : 0;
            uint32_t key = 0;
            int rc = bng_map_update(be_->ctx, config_, &key, &c, BNG_ANY);
            if (rc) return MapErr("failed to set config", rc);
        }
        return Nil();
    }
    Error Stop() {
        bindings_ = config_ = stats_ = ranges_ = -1;
        return Nil();
    }
    Error AddBinding(const MAC &mac, const IP &ipv4) { // :200-242
        if (mac.size() != 6) return Error("invalid MAC address");
        uint64_t key = ebpf::MACToUint64(mac);
        SubscriberBinding b;
        b.Mode = (uint8_t)mode_;
        if (!ipv4.empty() && To4(ipv4)) {
            b.IPv4Addr = be_ ? be_->AddrKey(ebpf::IPToUint32(ipv4)) : ebpf::IPToUint32(ipv4);
            b.IPv4Valid = 1;
        }
        if (bindings_ >= 0) {
            int rc = bng_map_update(be_->ctx, bindings_, &key, &b, BNG_ANY);
            if (rc) return MapErr("failed to update binding", rc);
        }
        std::lock_guard<std::mutex> g(mu_);
        subscribers_[key] = ipv4;
        return Nil();
    }
    Error AddBindingV6(const MAC &mac, const IP &ipv6) { // :245-282: lookup-modify-put
        if (mac.size() != 6) return Error("invalid MAC address");
        uint64_t key = ebpf::MACToUint64(mac);
        SubscriberBinding b;
        if (bindings_ >= 0) bng_map_lookup(be_->ctx, bindings_, &key, &b);
        if (ipv6.size() == 16) {
            memcpy(b.IPv6Addr, ipv6.data(), 16);
            b.IPv6Valid = 1;
        }
        b.Mode = (uint8_t)mode_;
        if (bindings_ >= 0) {
            int rc = bng_map_update(be_->ctx, bindings_, &key, &b, BNG_ANY);
            if (rc) return MapErr("failed to update binding", rc);
        }
        return Nil();
    }
    Error RemoveBinding(const MAC &mac) { // :285-301
        uint64_t key = ebpf::MACToUint64(mac);
        if (bindings_ >= 0) bng_map_delete(be_->ctx, bindings_, &key);
        std::lock_guard<std::mutex> g(mu_);
        subscribers_.erase(key);
        return Nil();
    }
    Error AddAllowedRange(const IP &network, int ones) { // :304-336 (*net.IPNet = address + prefix length)
        if (ranges_ < 0) return Error("ranges map not loaded");
        if (!To4(network)) return Error("IPv4 network required");
        struct {
            uint32_t Prefixlen, IP;
        } k{(uint32_t)ones, be_->AddrKey(ebpf::IPToUint32(network))};
        uint8_t one = 1;
        int rc = bng_map_update(be_->ctx, ranges_, &k, &one, BNG_ANY);
        return rc ? MapErr("failed to add range", rc) : Nil();
    }
    Result<Stats> GetStats() { // :339-352
        Result<Stats> r;
        if (stats_ < 0) {
            r.err = Error("stats map not loaded");
            return r;
        }
        uint32_t key = 0;
        Stats s;
        int rc = bng_map_lookup(be_->ctx, stats_, &key, &s);
        if (rc)
            r.err = MapErr("failed to get stats", rc);
        else
            r.value = s;
        return r;
    }
    int GetBindingCount() {
        std::lock_guard<std::mutex> g(mu_);
        return (int)subscribers_.size();
    }
    Error SetMode(Mode mode) { // :362-381
        mode_ = mode;
        if (config_ >= 0) {
            Config c;
            c.DefaultMode = (uint8_t)mode;
            c.LogViolations = cfg_.LogViolations ? 1 : 0;
            uint32_t key = 0;
            int rc = bng_map_update(be_->ctx, config_, &key, &c, BNG_ANY);
            if (rc) return MapErr("failed to update config", rc);
        }
        return Nil();
    }
    std::shared_ptr<Backend> backend() const { return be_; }

  private:
    Manager() = default;
    ManagerConfig cfg_;
    Mode mode_ = ModeDisabled;
    std::shared_ptr<Backend> be_;
    int bindings_ = -1, config_ = -1, stats_ = -1, ranges_ = -1;
    std::mutex mu_;
    std::map<uint64_t, IP> subscribers_;
};

} // namespace antispoof

// ===========================================================================
namespace qos {

#pragma pack(push, 1)
struct TokenBucket { // manager.go:19-26, bpf/qos_ratelimit.c:24-31 (32 bytes)
    uint64_t Tokens = 0, LastUpdate = 0, RateBPS = 0;
    uint32_t BurstBytes = 0;
    uint8_t Priority = 0, _pad[3] = {0, 0, 0};
};
struct QoSStats { // :29-34
    uint64_t PacketsPassed = 0, PacketsDropped = 0, BytesPassed = 0, BytesDropped = 0;
};
#pragma pack(pop)
static_assert(sizeof(TokenBucket) == 32 && sizeof(QoSStats) == 32, "ABI");

struct QoSPolicy { // pkg/radius/policy.go:12-20
    std::string Name;
    uint64_t DownloadBPS = 0, UploadBPS = 0;
    uint32_t BurstSize = 0;
    uint8_t Priority = 0;
};
inline std::vector<QoSPolicy> DefaultPolicies() { // pkg/radius/policy.go:70-128
    return {{"residential-50mbps", 50000000, 10000000, 1000000, 4},   {"residential-100mbps", 100000000, 20000000, 2000000, 4},
            {"residential-500mbps", 500000000, 50000000, 5000000, 4}, {"residential-1gbps", 1000000000, 100000000, 10000000, 4},
            {"business-100mbps", 100000000, 100000000, 2000000, 6},   {"business-1gbps", 1000000000, 1000000000, 10000000, 6},
            {"guest", 10000000, 5000000, 500000, 2},                  {"unlimited", 0, 0, 0, 4}};
}
struct SubscriberQoS { // manager.go:37-44
    IP Addr;
    uint64_t DownloadBPS = 0, UploadBPS = 0;
    uint32_t BurstBytes = 0;
    uint8_t Priority = 0;
    std::string PolicyName;
};
struct ManagerConfig {
    std::string Interface, BPFPath;
    std::shared_ptr<Backend> Backend_;
};

class Manager {
  public:
    static Result<std::shared_ptr<Manager>> NewManager(const ManagerConfig &cfg, std::vector<QoSPolicy> policies = {}) { // :69-86
        Result<std::shared_ptr<Manager>> r;
        if (cfg.Interface.empty()) {
            r.err = Error("interface required");
            return r;
        }
        auto m = std::shared_ptr<Manager>(new Manager());
        m->cfg_ = cfg;
        m->be_ = cfg.Backend_;
        m->havePolicies_ = !policies.empty();
        for (auto &p : policies) m->policies_[p.Name] = p;
        r.value = m;
        return r;
    }
    Error Start() { // :89-150
        if (!be_) be_ = Backend::Open();
        if (!be_->ctx) return Error("failed to load eBPF spec: " + be_->open_error);
        egress_ = be_->Map("qos_egress");
        if (egress_ < 0) return Error("qos_egress map not found");
        ingress_ = be_->Map("qos_ingress");
        if (ingress_ < 0) return Error("qos_ingress map not found");
        stats_ = be_->Map("qos_stats_map");
        return Nil();
    }
    Error Stop() {
        egress_ = ingress_ = stats_ = -1;
        return Nil();
    }
    // :167-245.  Burst defaulting: clamp(DownloadBPS/8, 64 KiB, 10 MiB) when BurstBytes == 0; the upload
    // bucket ALWAYS recomputes its burst from UploadBPS/8 with the same clamp; tokens start at burst, LastUpdate 0.
    static uint32_t defaultBurst(uint64_t bps) {
        uint32_t b = (uint32_t)(bps / 8);
        if (b < 65536) b = 65536;
        if (b > 10u * 1024 * 1024) b = 10u * 1024 * 1024;
        return b;
    }
    static TokenBucket egressBucket(const SubscriberQoS &q) {
        TokenBucket t;
        t.BurstBytes = q.BurstBytes ? q.BurstBytes : defaultBurst(q.DownloadBPS);
        t.Tokens = t.BurstBytes;
        t.RateBPS = q.DownloadBPS;
        t.Priority = q.Priority;
        return t;
    }
    static TokenBucket ingressBucket(const SubscriberQoS &q) {
        TokenBucket t;
        t.BurstBytes = defaultBurst(q.UploadBPS);
        t.Tokens = t.BurstBytes;
        t.RateBPS = q.UploadBPS;
        t.Priority = q.Priority;
        return t;
    }
    Error SetSubscriberQoS(const SubscriberQoS &q) {
        if (q.Addr.empty()) return Error("subscriber IP required");
        if (!To4(q.Addr)) return Error("IPv4 address required");
        uint32_t numeric = ebpf::IPToUint32(q.Addr);
        uint32_t key = be_ ? be_->AddrKey(numeric) : numeric;
        TokenBucket eg = egressBucket(q), in = ingressBucket(q);
        if (egress_ >= 0) {
            int rc = bng_map_update(be_->ctx, egress_, &key, &eg, BNG_ANY);
            if (rc) return MapErr("failed to set egress QoS", rc);
        }
        if (ingress_ >= 0) {
            int rc = bng_map_update(be_->ctx, ingress_, &key, &in, BNG_ANY);
            if (rc) return MapErr("failed to set ingress QoS", rc);
        }
        std::lock_guard<std::mutex> g(mu_);
        subscribers_[numeric] = q;
        return Nil();
    }
    Error SetSubscriberPolicy(const IP &ip, const std::string &policyName) { // :248-266
        if (!havePolicies_) return Error("policy manager not configured");
        auto it = policies_.find(policyName);
        if (it == policies_.end()) return Error("policy not found: " + policyName);
        SubscriberQoS q;
        q.Addr = ip;
        q.DownloadBPS = it->second.DownloadBPS;
        q.UploadBPS = it->second.UploadBPS;
        q.BurstBytes = it->second.BurstSize;
        q.Priority = it->second.Priority;
        q.PolicyName = policyName;
        return SetSubscriberQoS(q);
    }
    Error RemoveSubscriberQoS(const IP &ip) { // :269-295
        if (!To4(ip)) return Error("IPv4 address required");
        uint32_t numeric = ebpf::IPToUint32(ip);
        uint32_t key = be_ ? be_->AddrKey(numeric) : numeric;
        if (egress_ >= 0) bng_map_delete(be_->ctx, egress_, &key);
        if (ingress_ >= 0) bng_map_delete(be_->ctx, ingress_, &key);
        std::lock_guard<std::mutex> g(mu_);
        subscribers_.erase(numeric);
        return Nil();
    }
    Result<QoSStats> GetStats() { // :298-313
        Result<QoSStats> r;
        if (stats_ < 0) {
            r.err = Error("stats map not loaded");
            return r;
        }
        uint32_t key = 0;
        QoSStats s;
        int rc = bng_map_lookup(be_->ctx, stats_, &key, &s);
        if (rc)
            r.err = MapErr("failed to get stats", rc);
        else
            r.value = s;
        return r;
    }
    int GetSubscriberCount() {
        std::lock_guard<std::mutex> g(mu_);
        return (int)subscribers_.size();
    }
    std::shared_ptr<Backend> backend() const { return be_; }

  private:
    Manager() = default;
    ManagerConfig cfg_;
    std::shared_ptr<Backend> be_;
    bool havePolicies_ = false;
    std::map<std::string, QoSPolicy> policies_;
    int egress_ = -1, ingress_ = -1, stats_ = -1;
    std::mutex mu_;
    std::map<uint32_t, SubscriberQoS> subscribers_;
};

} // namespace qos

// ===========================================================================
namespace nat {

// flags / events / ALG types, manager.go:17-44
enum : uint32_t {
    NATFlagEIMEnabled = 0x01, NATFlagEIFEnabled = 0x02, NATFlagHairpinEnabled = 0x04, NATFlagALGFTP = 0x08,
    NATFlagALGSIP = 0x10, NATFlagPortParity = 0x20, NATFlagPortContiguity = 0x40
};
enum : uint32_t {
    NATLogSessionCreate = 1, NATLogSessionDelete = 2, NATLogPortBlockAssign = 3, NATLogPortBlockRelease = 4,
    NATLogPortExhaustion = 5, NATLogHairpin = 6, NATLogALGTrigger = 7
};
enum : uint8_t { ALGTypeFTP = 1, ALGTypeSIP = 2, ALGTypeRTSP = 3 };

// The C layouts are the contract (bpf/nat44.c:92-213); the reference's Go mirrors of port_block /
// nat_session / nat_log_entry no longer match them (SURVEY.md §7.3-4) and are NOT reproduced.
#pragma pack(push, 1)
struct PortBlock { // bpf/nat44.c:144-155 (32 bytes)
    uint32_t PublicIP = 0;
    uint16_t PortStart = 0, PortEnd = 0;
    uint32_t NextPort = 0, PortsInUse = 0;
    uint64_t AllocatedAt = 0;
    uint32_t SubscriberID = 0;
    uint8_t BlockSizeLog2 = 0, Flags = 0, _pad[2] = {0, 0};
};
struct SubscriberNAT { // :158-164 (64 bytes)
    PortBlock Block;
    uint64_t SessionsActive = 0, SessionsTotal = 0, BytesOut = 0, BytesIn = 0;
};
struct NATKey { // :92-99
    uint32_t SrcIP = 0, DstIP = 0;
    uint16_t SrcPort = 0, DstPort = 0;
    uint8_t Protocol = 0, _pad[3] = {0, 0, 0};
};
struct NATSession { // :123-141 (80 bytes)
    uint32_t NATIP;
    uint16_t NATPort, OrigPort;
    uint32_t OrigIP, DestIP;
    uint16_t DestPort, _pad1;
    uint32_t _ipad;
    uint64_t LastSeen, Created, PacketsOut, PacketsIn, BytesOut, BytesIn;
    uint8_t State, Protocol, Flags, IsHairpin;
    uint32_t _tpad;
};
struct EIMKey { // :104-109
    uint32_t InternalIP = 0;
    uint16_t InternalPort = 0;
    uint8_t Protocol = 0, _pad = 0;
};
struct EIMMapping { // :112-120
    uint32_t ExternalIP;
    uint16_t ExternalPort, _pad;
    uint64_t Created, LastUsed;
    uint32_t RefCount, Flags;
};
struct NATStats { // :176-190 (104 bytes)
    uint64_t PacketsSNAT = 0, PacketsDNAT = 0, PacketsHairpin = 0, PacketsDropped = 0, PacketsPassed = 0, SessionsCreated = 0,
             SessionsExpired = 0, PortExhaustion = 0, EIMHits = 0, EIMMisses = 0, ALGTriggers = 0, ConntrackLookups = 0,
             ConntrackHits = 0;
};
struct NATConfig { // :271-277
    uint32_t Flags = 0;
    uint16_t PortRangeStart = 0, PortRangeEnd = 0;
    uint32_t DefaultPortsPerSub = 0, _pad = 0;
};
struct ALGConfig { // :208-213
    uint16_t Port = 0;
    uint8_t Protocol = 0, ALGType = 0;
    uint32_t Flags = 0;
};
struct LogEntry { // nat_log_entry, :193-205 (40 bytes)
    uint64_t Timestamp;
    uint32_t EventType, SubscriberID, PrivateIP, PublicIP;
    uint16_t PrivatePort, PublicPort;
    uint32_t DestIP;
    uint16_t DestPort;
    uint8_t Protocol, Flags;
    uint32_t _tpad;
};
#pragma pack(pop)
static_assert(sizeof(PortBlock) == 32 && sizeof(SubscriberNAT) == 64 && sizeof(NATKey) == 16 && sizeof(NATSession) == 80, "ABI");
static_assert(sizeof(EIMKey) == 8 && sizeof(EIMMapping) == 32 && sizeof(NATStats) == 104 && sizeof(NATConfig) == 16, "ABI");
static_assert(sizeof(ALGConfig) == 8 && sizeof(LogEntry) == 40, "ABI");

inline int log2(int n) { // manager.go:837-844
    int r = 0;
    while (n > 1) {
        n >>= 1;
        r++;
    }
    return r;
}

struct PoolEntry { // manager.go:151-158
    IP PublicIP;
    int TotalPorts = 0, PortsPerSub = 0, Subscribers = 0, MaxSubscribers = 0;
    uint32_t Flags = 0;
};
struct Allocation { // :161-169
    IP PrivateIP, PublicIP;
    uint16_t PortStart = 0, PortEnd = 0;
    int PoolIndex = 0;
    uint32_t SubscriberID = 0;
    uint64_t AllocatedAtNs = 0;
};
struct ManagerConfig { // :172-200
    std::string Interface, BPFPath;
    int PortsPerSubscriber = 0, PortRangeStart = 0, PortRangeEnd = 0;
    bool EnableEIM = false, EnableEIF = false, EnableHairpin = false, EnableFTPALG = false, EnableSIPALG = false,
         EnablePortParity = false, EnablePortContiguity = false, EnableLogging = false;
    std::shared_ptr<Backend> Backend_;
};

class Manager {
  public:
    static Result<std::shared_ptr<Manager>> NewManager(const ManagerConfig &cfg) { // :253-292
        Result<std::shared_ptr<Manager>> r;
        if (cfg.Interface.empty()) {
            r.err = Error("interface required");
            return r;
        }
        auto m = std::shared_ptr<Manager>(new Manager());
        m->cfg_ = cfg;
        m->be_ = cfg.Backend_;
        m->portsPerSubscriber_ = cfg.PortsPerSubscriber ? cfg.PortsPerSubscriber : 1024;
        m->portRangeStart_ = cfg.PortRangeStart ? cfg.PortRangeStart : 1024;
        m->portRangeEnd_ = cfg.PortRangeEnd ? cfg.PortRangeEnd : 65535;
        r.value = m;
        return r;
    }
    uint32_t buildFlags() const { // :371-395
        uint32_t f = 0;
        if (cfg_.EnableEIM) f |= NATFlagEIMEnabled;
        if (cfg_.EnableEIF) f |= NATFlagEIFEnabled;
        if (cfg_.EnableHairpin) f |= NATFlagHairpinEnabled;
        if (cfg_.EnableFTPALG) f |= NATFlagALGFTP;
        if (cfg_.EnableSIPALG) f |= NATFlagALGSIP;
        if (cfg_.EnablePortParity) f |= NATFlagPortParity;
        if (cfg_.EnablePortContiguity) f |= NATFlagPortContiguity;
        return f;
    }
    Error AddPublicIP(const IP &ip) { // :310-350
        if (!To4(ip)) return Error("IPv4 address required");
        std::lock_guard<std::mutex> g(poolMu_);
        PoolEntry e;
        e.PublicIP = IP(To4(ip), To4(ip) + 4);
        e.TotalPorts = portRangeEnd_ - portRangeStart_ + 1;
        e.PortsPerSub = portsPerSubscriber_;
        e.MaxSubscribers = e.TotalPorts / portsPerSubscriber_;
        e.Flags = buildFlags();
        pool_.push_back(e);
        if (hairpinIPs_ >= 0 && cfg_.EnableHairpin) {
            uint32_t k = be_->AddrKey(ebpf::IPToUint32(ip));
            uint8_t one = 1;
            bng_map_update(be_->ctx, hairpinIPs_, &k, &one, BNG_ANY);
        }
        return Nil();
    }
    Error AddPublicIPRange(const IP &startIP, const IP &endIP) { // :353-368
        uint32_t s = ebpf::IPToUint32(startIP), e = ebpf::IPToUint32(endIP);
        if (s > e) return Error("start IP must be less than or equal to end IP");
        for (uint64_t a = s; a <= e; a++) {
            Error err = AddPublicIP(ebpf::Uint32ToIP((uint32_t)a));
            if (err) return Error("failed to add IP: " + err.what());
        }
        return Nil();
    }
    // AllocateNAT, :398-494: first pool entry with Subscribers < MaxSubscribers; the block is
    // [rangeStart + Subscribers*pps, +pps-1]; sequential subscriber ids from 1; writes subscriber_nat.
    Result<Allocation> AllocateNAT(const IP &privateIP) {
        Result<Allocation> r;
        if (!To4(privateIP)) {
            r.err = Error("IPv4 address required");
            return r;
        }
        uint32_t privKey = ebpf::IPToUint32(privateIP);
        {
            std::lock_guard<std::mutex> g(allocMu_);
            auto it = allocations_.find(privKey);
            if (it != allocations_.end()) {
                r.value = it->second;
                return r;
            }
        }
        std::lock_guard<std::mutex> g(poolMu_);
        PoolEntry *sel = nullptr;
        int idx = 0;
        for (size_t i = 0; i < pool_.size(); i++)
            if (pool_[i].Subscribers < pool_[i].MaxSubscribers) {
                sel = &pool_[i];
                idx = (int)i;
                break;
            }
        if (!sel) {
            r.err = Error("NAT pool exhausted: no available public IPs");
            return r;
        }
        uint16_t portStart = (uint16_t)(portRangeStart_ + sel->Subscribers * portsPerSubscriber_);
        uint16_t portEnd = (uint16_t)(portStart + (uint16_t)portsPerSubscriber_ - 1);
        uint32_t sid = getOrCreateSubscriberID(privKey);
        Allocation a;
        a.PrivateIP = IP(To4(privateIP), To4(privateIP) + 4);
        a.PublicIP = sel->PublicIP;
        a.PortStart = portStart;
        a.PortEnd = portEnd;
        a.PoolIndex = idx;
        a.SubscriberID = sid;
        a.AllocatedAtNs = (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(
                              std::chrono::system_clock::now().time_since_epoch()).count();
        if (subscriberNAT_ >= 0) {
            SubscriberNAT sn;
            sn.Block.PublicIP = be_->AddrKey(ebpf::IPToUint32(sel->PublicIP));
            sn.Block.PortStart = portStart;
            sn.Block.PortEnd = portEnd;
            sn.Block.NextPort = portStart;
            sn.Block.AllocatedAt = a.AllocatedAtNs;
            sn.Block.SubscriberID = sid;
            sn.Block.BlockSizeLog2 = (uint8_t)log2(portsPerSubscriber_);
            uint32_t k = be_->AddrKey(privKey);
            int rc = bng_map_update(be_->ctx, subscriberNAT_, &k, &sn, BNG_ANY);
            if (rc) {
                r.err = MapErr("failed to update eBPF map", rc);
                return r;
            }
        }
        {
            std::lock_guard<std::mutex> g2(allocMu_);
            allocations_[privKey] = a;
        }
        sel->Subscribers++;
        r.value = a;
        return r;
    }
    Error DeallocateNAT(const IP &privateIP) { // :497-539 (Subscribers-- can make later blocks overlap: kept)
        if (!To4(privateIP)) return Error("IPv4 address required");
        uint32_t privKey = ebpf::IPToUint32(privateIP);
        Allocation a;
        {
            std::lock_guard<std::mutex> g(allocMu_);
            auto it = allocations_.find(privKey);
            if (it == allocations_.end()) return Nil();
            a = it->second;
            allocations_.erase(it);
        }
        if (subscriberNAT_ >= 0) {
            uint32_t k = be_->AddrKey(privKey);
            bng_map_delete(be_->ctx, subscriberNAT_, &k);
        }
        std::lock_guard<std::mutex> g(poolMu_);
        if (a.PoolIndex < (int)pool_.size()) pool_[a.PoolIndex].Subscribers--;
        return Nil();
    }
    // Not in the reference: DeallocateNAT leaves the subscribers' sessions, reverse entries and EIM mappings on the
    // dataplane until they expire, and the next holder of the address inherits them.  One bng_nat_flush pass removes
    // them.  Call it before DeallocateNAT, so that the NAT log records still carry the subscriber id.
    // removed_out (may be null): sessions, reverse entries, EIM mappings removed.
    Error FlushSessions(const std::vector<IP> &privateIPs, uint64_t now_ns, uint64_t removed_out[3] = nullptr) {
        if (!be_ || !be_->ctx) return Error("dataplane not open");
        std::vector<uint32_t> keys;
        keys.reserve(privateIPs.size());
        for (const IP &ip : privateIPs) {
            if (!To4(ip)) return Error("IPv4 address required");
            keys.push_back(be_->AddrKey(ebpf::IPToUint32(ip)));
        }
        return MapErr("bng_nat_flush", bng_nat_flush(be_->ctx, keys.data(), keys.size(), now_ns, removed_out));
    }
    Error ConfigureALG(uint16_t port, uint8_t protocol, uint8_t algType, bool enabled) { // :542-560
        if (algPorts_ < 0) return Error("ALG map not loaded");
        uint32_t key = ((uint32_t)port << 16) | protocol;
        if (enabled) {
            ALGConfig c;
            c.Port = port;
            c.Protocol = protocol;
            c.ALGType = algType;
            return MapErr("update", bng_map_update(be_->ctx, algPorts_, &key, &c, BNG_ANY));
        }
        return MapErr("delete", bng_map_delete(be_->ctx, algPorts_, &key));
    }
    Error Start() { // :563-652
        if (!be_) be_ = Backend::Open();
        if (!be_->ctx) return Error("failed to load eBPF spec: " + be_->open_error);
        subscriberNAT_ = be_->Map("subscriber_nat");
        if (subscriberNAT_ < 0) return Error("subscriber_nat map not found");
        natSessions_ = be_->Map("nat_sessions");
        natReverse_ = be_->Map("nat_reverse");
        natPool_ = be_->Map("nat_pool");
        natStats_ = be_->Map("nat_stats_map");
        natConfigMap_ = be_->Map("nat_config_map");
        eimTable_ = be_->Map("eim_table");
        hairpinIPs_ = be_->Map("hairpin_ips");
        algPorts_ = be_->Map("alg_ports");
        natLogRB_ = be_->Map("nat_log_rb");
        if (natConfigMap_ >= 0) {
            NATConfig c;
            c.Flags = buildFlags();
            c.PortRangeStart = (uint16_t)portRangeStart_;
            c.PortRangeEnd = (uint16_t)portRangeEnd_;
            c.DefaultPortsPerSub = (uint32_t)portsPerSubscriber_;
            uint32_t key = 0;
            bng_map_update(be_->ctx, natConfigMap_, &key, &c, BNG_ANY);
        }
        if (cfg_.EnableFTPALG) ConfigureALG(21, 6, ALGTypeFTP, true);
        if (cfg_.EnableSIPALG) {
            ConfigureALG(5060, 17, ALGTypeSIP, true);
            ConfigureALG(5060, 6, ALGTypeSIP, true);
        }
        return Nil();
    }
    Error Stop() {
        subscriberNAT_ = natSessions_ = natReverse_ = natPool_ = natStats_ = natConfigMap_ = eimTable_ = hairpinIPs_ = algPorts_ =
            natLogRB_ = -1;
        return Nil();
    }
    Result<NATStats> GetStats() { // :721-734
        Result<NATStats> r;
        if (natStats_ < 0) {
            r.err = Error("stats map not loaded");
            return r;
        }
        uint32_t key = 0;
        NATStats s;
        int rc = bng_map_lookup(be_->ctx, natStats_, &key, &s);
        if (rc)
            r.err = MapErr("failed to get stats", rc);
        else
            r.value = s;
        return r;
    }
    int GetAllocationCount() {
        std::lock_guard<std::mutex> g(allocMu_);
        return (int)allocations_.size();
    }
    std::vector<PoolEntry> GetPoolStats() {
        std::lock_guard<std::mutex> g(poolMu_);
        return pool_;
    }
    std::optional<Allocation> GetAllocation(const IP &privateIP) { // :754-764
        if (!To4(privateIP)) return std::nullopt;
        std::lock_guard<std::mutex> g(allocMu_);
        auto it = allocations_.find(ebpf::IPToUint32(privateIP));
        if (it == allocations_.end()) return std::nullopt;
        return it->second;
    }
    Result<EIMMapping> GetEIMMapping(const IP &internalIP, uint16_t internalPort, uint8_t protocol) { // :767-784
        Result<EIMMapping> r;
        if (eimTable_ < 0) {
            r.err = Error("EIM table not loaded");
            return r;
        }
        EIMKey k;
        k.InternalIP = be_->AddrKey(ebpf::IPToUint32(internalIP));
        k.InternalPort = internalPort;
        k.Protocol = protocol;
        EIMMapping m{};
        int rc = bng_map_lookup(be_->ctx, eimTable_, &k, &m);
        if (rc)
            r.err = MapErr("lookup", rc);
        else
            r.value = m;
        return r;
    }
    Result<NATSession> LookupSession(const IP &srcIP, const IP &dstIP, uint16_t srcPort, uint16_t dstPort, uint8_t protocol) {
        Result<NATSession> r; // :787-816
        if (natSessions_ < 0) {
            r.err = Error("sessions map not loaded");
            return r;
        }
        NATKey k;
        k.SrcIP = be_->AddrKey(ebpf::IPToUint32(srcIP));
        k.DstIP = be_->AddrKey(ebpf::IPToUint32(dstIP));
        k.SrcPort = srcPort;
        k.DstPort = dstPort;
        k.Protocol = protocol;
        NATSession s{};
        int rc = bng_map_lookup(be_->ctx, natSessions_, &k, &s);
        if (rc)
            r.err = MapErr("lookup", rc);
        else
            r.value = s;
        return r;
    }
    // The reference's ring-buffer reader is a placeholder (manager.go:682-696); this drains nat_log_rb.
    std::vector<LogEntry> DrainLog(size_t max = 1 << 16) {
        std::vector<LogEntry> out;
        if (natLogRB_ < 0) return out;
        out.resize(max);
        uint64_t n = 0;
        if (bng_events_drain(be_->ctx, natLogRB_, out.data(), max, &n)) n = 0;
        out.resize(n);
        return out;
    }
    std::shared_ptr<Backend> backend() const { return be_; }

  private:
    Manager() = default;
    uint32_t getOrCreateSubscriberID(uint32_t privateIP) { // :295-307
        std::lock_guard<std::mutex> g(idMu_);
        auto it = subscriberIDs_.find(privateIP);
        if (it != subscriberIDs_.end()) return it->second;
        uint32_t id = nextSubscriberID_++;
        subscriberIDs_[privateIP] = id;
        return id;
    }
    ManagerConfig cfg_;
    std::shared_ptr<Backend> be_;
    int portsPerSubscriber_ = 1024, portRangeStart_ = 1024, portRangeEnd_ = 65535;
    int subscriberNAT_ = -1, natSessions_ = -1, natReverse_ = -1, natPool_ = -1, natStats_ = -1, natConfigMap_ = -1,
        eimTable_ = -1, hairpinIPs_ = -1, algPorts_ = -1, natLogRB_ = -1;
    std::mutex poolMu_, allocMu_, idMu_;
    std::vector<PoolEntry> pool_;
    std::map<uint32_t, Allocation> allocations_;
    uint32_t nextSubscriberID_ = 1;
    std::map<uint32_t, uint32_t> subscriberIDs_;
};

} // namespace nat
} // namespace bng
