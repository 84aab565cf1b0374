// bng_dhcp_slow.hpp — the DHCPv4 *slow path* of the reference, restated in C++ (BASELINE.json config #1,
// SURVEY.md §8d: "CPU only, plumbing").  It is the only per-packet Go code of the reference and the
// caller on the far side of the fast path: what it decides is mirrored into the subscriber_pools /
// ip_pools maps through ebpf::Loader, and from then on the GPU's dhcp_fastpath kernel answers.
//
// Restates (nothing copied, Go -> C++):
//   bng::dhcp::Pool         pkg/dhcp/pool.go:23-39,56-224   (NewPool, generateAvailableIPs, Allocate, Release, ...)
//   bng::dhcp::PoolManager  pkg/dhcp/pool.go:233-360        (AddPool mirrors the pool into ip_pools)
//   bng::dhcp::Server       pkg/dhcp/server.go:302-383 (handleDHCP dispatch), :398-553 (handleDiscover),
//                           :556-860 (handleRequest, local-pool branch), :1043-1054 (buildNAK),
//                           :1057-1097 (updateFastPathCache)
// Out of scope, as in the survey: RADIUS authentication, the Nexus / HTTP allocator branches, option 82
// bookkeeping beyond carrying it, RELEASE / DECLINE / INFORM, accounting.
//
// The reply encoder stands in for github.com/insomniacslk/dhcp v0.0.0-20231206064809-8c70d406f6d2
// (go.mod:8), which is not vendored in /root/reference: NewReplyFromRequest() + ToBytes() are restated from
// RFC 2131 / RFC 1542 and that library's documented behaviour (BOOTREPLY, xid / flags / htype / chaddr /
// giaddr copied from the request, options emitted in ascending code order, option 255, padded to the
// 300-byte BOOTP minimum).  PARITY UNPINNED for this file: there is no Go toolchain here to run the
// reference's pkg/dhcp tests; tests/host/test_host.cpp re-derives pool_test.go's expectations instead.
#pragma once

#include <deque>
#include <functional>

#include "bng_host.hpp"

namespace bng {
namespace dhcp {

using Clock = std::function<int64_t()>; // seconds since the epoch (time.Now().Unix())
inline int64_t WallClock() {
    return std::chrono::duration_cast<std::chrono::seconds>(std::chrono::system_clock::now().time_since_epoch()).count();
}

enum MessageType : uint8_t { Discover = 1, Offer = 2, Request = 3, Decline = 4, Ack = 5, Nak = 6, Release = 7, Inform = 8 };
enum Option : uint8_t {
    OptSubnetMask = 1, OptRouter = 3, OptDNS = 6, OptHostName = 12, OptRequestedIP = 50, OptLeaseTime = 51, OptMessageType = 53,
    OptServerID = 54, OptParamList = 55, OptClientID = 61, OptRelayAgentInfo = 82, OptEnd = 255,
};

// A DHCPv4 message (RFC 2131 figure 1); addresses as big-endian numerics like ebpf::IPToUint32.
struct Message {
    uint8_t op = 1, htype = 1, hlen = 6, hops = 0;
    uint32_t xid = 0;
    uint16_t secs = 0, flags = 0;
    uint32_t ciaddr = 0, yiaddr = 0, siaddr = 0, giaddr = 0;
    uint8_t chaddr[16] = {0};
    std::map<uint8_t, std::vector<uint8_t>> options;

    MAC ClientHWAddr() const { return MAC(chaddr, chaddr + (hlen <= 16 ? hlen : 16)); }
    int Type() const {
        auto it = options.find(OptMessageType);
        return it != options.end() && it->second.size() == 1 ? it->second[0] : 0;
    }
    uint32_t RequestedIP() const {
        auto it = options.find(OptRequestedIP);
        if (it == options.end() || it->second.size() != 4) return 0;
        const auto &v = it->second;
        return ((uint32_t)v[0] << 24) | ((uint32_t)v[1] << 16) | ((uint32_t)v[2] << 8) | v[3];
    }
    void SetIPOption(uint8_t code, uint32_t ip) { options[code] = {(uint8_t)(ip >> 24), (uint8_t)(ip >> 16), (uint8_t)(ip >> 8), (uint8_t)ip}; }

    static Result<Message> Parse(const uint8_t *p, size_t n) {
        Result<Message> r;
        if (n < 240) {
            r.err = Error("dhcpv4: packet shorter than the BOOTP header");
            return r;
        }
        static const uint8_t cookie[4] = {0x63, 0x82, 0x53, 0x63};
        if (memcmp(p + 236, cookie, 4)) {
            r.err = Error("dhcpv4: bad magic cookie");
            return r;
        }
        Message m;
        m.op = p[0], m.htype = p[1], m.hlen = p[2], m.hops = p[3];
        auto be32 = [&](size_t o) { return ((uint32_t)p[o] << 24) | ((uint32_t)p[o + 1] << 16) | ((uint32_t)p[o + 2] << 8) | p[o + 3]; };
        m.xid = be32(4);
        m.secs = (uint16_t)((p[8] << 8) | p[9]);
        m.flags = (uint16_t)((p[10] << 8) | p[11]);
        m.ciaddr = be32(12), m.yiaddr = be32(16), m.siaddr = be32(20), m.giaddr = be32(24);
        memcpy(m.chaddr, p + 28, 16);
        for (size_t o = 240; o < n;) {
            uint8_t code = p[o++];
            if (code == 0) continue;
            if (code == OptEnd) break;
            if (o >= n) break;
            uint8_t len = p[o++];
            if (o + len > n) break;
            auto &v = m.options[code]; // a repeated option concatenates (RFC 3396)
            v.insert(v.end(), p + o, p + o + len);
            o += len;
        }
        r.value = std::move(m);
        return r;
    }
    std::vector<uint8_t> ToBytes() const {
        std::vector<uint8_t> b(240, 0);
        b[0] = op, b[1] = htype, b[2] = hlen, b[3] = hops;
        auto put32 = [&](size_t o, uint32_t v) { b[o] = (uint8_t)(v >> 24), b[o + 1] = (uint8_t)(v >> 16), b[o + 2] = (uint8_t)(v >> 8), b[o + 3] = (uint8_t)v; };
        put32(4, xid);
        b[8] = (uint8_t)(secs >> 8), b[9] = (uint8_t)secs, b[10] = (uint8_t)(flags >> 8), b[11] = (uint8_t)flags;
        put32(12, ciaddr), put32(16, yiaddr), put32(20, siaddr), put32(24, giaddr);
        memcpy(&b[28], chaddr, 16);
        b[236] = 0x63, b[237] = 0x82, b[238] = 0x53, b[239] = 0x63;
        for (const auto &kv : options) { // std::map iterates in ascending code order
            size_t off = 0;
            do { // options longer than 255 bytes are split
                size_t n = kv.second.size() - off;
                if (n > 255) n = 255;
                b.push_back(kv.first);
                b.push_back((uint8_t)n);
                b.insert(b.end(), kv.second.begin() + off, kv.second.begin() + off + n);
                off += n;
            } while (off < kv.second.size());
        }
        b.push_back(OptEnd);
        if (b.size() < 300) b.resize(300, 0); // BOOTP minimum (RFC 1542 §2.1)
        return b;
    }
    // dhcpv4.NewReplyFromRequest: a BOOTREPLY that echoes what identifies the exchange
    static Message ReplyTo(const Message &req) {
        Message r;
        r.op = 2;
        r.htype = req.htype, r.hlen = req.hlen;
        r.xid = req.xid;
        r.flags = req.flags;
        r.giaddr = req.giaddr;
        memcpy(r.chaddr, req.chaddr, 16);
        for (uint8_t code : {(uint8_t)OptRelayAgentInfo, (uint8_t)OptClientID}) { // copied when present (RFC 3046, RFC 6842)
            auto it = req.options.find(code);
            if (it != req.options.end()) r.options[code] = it->second;
        }
        return r;
    }
};

// --------------------------------------------------------------------------- pkg/dhcp/pool.go
struct PoolConfig { // :42-54
    uint32_t ID = 0;
    std::string Name;
    std::string Network; // CIDR
    std::string Gateway;
    std::vector<std::string> DNSServers;
    int64_t LeaseTimeSec = 0;
    uint8_t ClientClass = 0;
    uint32_t VlanID = 0;
    int ReservedStart = 0, ReservedEnd = 0;
};
struct PoolStats { // :216-224
    int Total = 0, Allocated = 0, Available = 0, Unavailable = 0;
};

inline bool ParseIPv4(const std::string &s, uint32_t *out) {
    unsigned a, b, c, d;
    char tail;
    if (sscanf(s.c_str(), "%u.%u.%u.%u%c", &a, &b, &c, &d, &tail) != 4 || a > 255 || b > 255 || c > 255 || d > 255) return false;
    *out = (a << 24) | (b << 16) | (c << 8) | d;
    return true;
}

class Pool {
  public:
    uint32_t ID = 0;
    std::string Name;
    uint32_t Network = 0; // network address (masked), big-endian numeric
    int PrefixLen = 0;
    uint32_t Gateway = 0, SubnetMask = 0;
    std::vector<uint32_t> DNSServers;
    int64_t LeaseTimeSec = 0;
    uint8_t ClientClass = 0;
    uint32_t VlanID = 0;

    static Result<std::shared_ptr<Pool>> New(const PoolConfig &cfg) { // NewPool, :57-96
        Result<std::shared_ptr<Pool>> r;
        auto slash = cfg.Network.find('/');
        uint32_t addr = 0;
        int ones = -1;
        if (slash != std::string::npos) ones = atoi(cfg.Network.c_str() + slash + 1);
        if (slash == std::string::npos || !ParseIPv4(cfg.Network.substr(0, slash), &addr) || ones < 0 || ones > 32) {
            r.err = Error("invalid network CIDR: " + cfg.Network);
            return r;
        }
        auto p = std::make_shared<Pool>();
        if (!ParseIPv4(cfg.Gateway, &p->Gateway)) {
            r.err = Error("invalid gateway IP: " + cfg.Gateway);
            return r;
        }
        for (const auto &d : cfg.DNSServers) {
            uint32_t ip;
            if (!ParseIPv4(d, &ip)) {
                r.err = Error("invalid DNS server IP: " + d);
                return r;
            }
            p->DNSServers.push_back(ip);
        }
        p->ID = cfg.ID, p->Name = cfg.Name, p->PrefixLen = ones;
        p->SubnetMask = ones == 0 ? 0 : 0xFFFFFFFFu << (32 - ones);
        p->Network = addr & p->SubnetMask;
        p->LeaseTimeSec = cfg.LeaseTimeSec, p->ClientClass = cfg.ClientClass, p->VlanID = cfg.VlanID;
        p->generateAvailable(cfg.ReservedStart, cfg.ReservedEnd);
        r.value = p;
        return r;
    }
    Result<uint32_t> Allocate(uint64_t mac) { // :146-167: an existing allocation is returned again; else the list's head
        std::lock_guard<std::mutex> g(mu_);
        Result<uint32_t> r;
        auto it = allocated_.find(mac);
        if (it != allocated_.end()) {
            r.value = it->second;
            return r;
        }
        if (available_.empty()) {
            r.err = Error("pool " + Name + " exhausted");
            return r;
        }
        uint32_t ip = available_.front();
        available_.pop_front();
        allocated_[mac] = ip;
        r.value = ip;
        return r;
    }
    void Release(uint32_t ip) { // :170-184: back to the END of the list
        std::lock_guard<std::mutex> g(mu_);
        for (auto it = allocated_.begin(); it != allocated_.end(); ++it)
            if (it->second == ip) {
                allocated_.erase(it);
                available_.push_back(ip);
                return;
            }
    }
    // The allocation of `mac`, if it is `ip`, back to the end of the list; false: the address is not (or no longer) this
    // client's, and whoever holds it now keeps it.
    bool ReleaseFor(uint64_t mac, uint32_t ip) {
        std::lock_guard<std::mutex> g(mu_);
        auto it = allocated_.find(mac);
        if (it == allocated_.end() || it->second != ip) return false;
        allocated_.erase(it);
        available_.push_back(ip);
        return true;
    }
    bool Contains(uint32_t ip) const { return (ip & SubnetMask) == Network; } // :187-189
    PoolStats Stats() { // :205-214
        std::lock_guard<std::mutex> g(mu_);
        PoolStats s;
        s.Allocated = (int)allocated_.size(), s.Available = (int)available_.size(), s.Unavailable = (int)unavailable_.size();
        s.Total = s.Allocated + s.Available + s.Unavailable;
        return s;
    }
    void MarkUnavailable(uint32_t ip) { // :192-203
        std::lock_guard<std::mutex> g(mu_);
        unavailable_[ip] = true;
        for (auto it = available_.begin(); it != available_.end(); ++it)
            if (*it == ip) {
                available_.erase(it);
                break;
            }
    }

  private:
    void generateAvailable(int reservedStart, int reservedEnd) { // :99-142
        int hostBits = 32 - PrefixLen;
        long numHosts = (hostBits >= 31 ? (1L << 31) : (1L << hostBits)) - 2; // network and broadcast excluded
        if (numHosts <= 0) return;
        for (long i = 1; i <= numHosts; i++) {
            if (i <= reservedStart) continue;
            if (i > numHosts - reservedEnd) continue;
            uint32_t ip = Network + (uint32_t)i;
            if (ip == Gateway) continue;
            available_.push_back(ip);
        }
    }
    std::map<uint64_t, uint32_t> allocated_;
    std::deque<uint32_t> available_;
    std::map<uint32_t, bool> unavailable_;
    std::mutex mu_;
};

class PoolManager { // :233-360
  public:
    explicit PoolManager(ebpf::Loader *loader = nullptr) : loader_(loader) {}
    Error AddPool(std::shared_ptr<Pool> pool) { // :248-297
        std::lock_guard<std::mutex> g(mu_);
        if (pools_.count(pool->ID)) return Error("pool " + std::to_string(pool->ID) + " already exists");
        pools_[pool->ID] = pool;
        if (pools_.size() == 1) defaultPoolID_ = pool->ID; // the first pool becomes the default
        if (loader_) {                                     // mirrored into the fast path's ip_pools map
            ebpf::IPPool p;
            p.Network = pool->Network;
            p.PrefixLen = (uint8_t)pool->PrefixLen;
            p.Gateway = pool->Gateway;
            p.DNSPrimary = pool->DNSServers.size() > 0 ? pool->DNSServers[0] : 0;
            p.DNSSecondary = pool->DNSServers.size() > 1 ? pool->DNSServers[1] : 0;
            p.LeaseTime = (uint32_t)pool->LeaseTimeSec;
            lastSyncError_ = loader_->AddPool(pool->ID, p); // the reference only logs a failure here
        }
        return Nil();
    }
    Error RemovePool(uint32_t id) { // :300-315
        std::lock_guard<std::mutex> g(mu_);
        if (!pools_.count(id)) return Error("pool " + std::to_string(id) + " not found");
        pools_.erase(id);
        if (loader_) loader_->RemovePool(id);
        return Nil();
    }
    std::shared_ptr<Pool> GetPool(uint32_t id) {
        std::lock_guard<std::mutex> g(mu_);
        auto it = pools_.find(id);
        return it == pools_.end() ? nullptr : it->second;
    }
    std::shared_ptr<Pool> ClassifyClient(uint64_t /*mac*/) { // :323-341: the default pool, else any pool
        std::lock_guard<std::mutex> g(mu_);
        auto it = pools_.find(defaultPoolID_);
        if (it != pools_.end()) return it->second;
        return pools_.empty() ? nullptr : pools_.begin()->second;
    }
    Error SetDefaultPool(uint32_t id) { // :344-353
        std::lock_guard<std::mutex> g(mu_);
        if (!pools_.count(id)) return Error("pool " + std::to_string(id) + " not found");
        defaultPoolID_ = id;
        return Nil();
    }
    const Error &LastSyncError() const { return lastSyncError_; }

  private:
    std::map<uint32_t, std::shared_ptr<Pool>> pools_;
    std::mutex mu_;
    ebpf::Loader *loader_;
    uint32_t defaultPoolID_ = 0;
    Error lastSyncError_;
};

// --------------------------------------------------------------------------- pkg/dhcp/server.go
struct Lease { // :81-103 (the fields the local path uses)
    uint64_t MAC = 0;
    uint32_t IP = 0, PoolID = 0;
    int64_t ExpiresAt = 0;
    std::string Hostname;
    uint16_t STag = 0, CTag = 0;
    std::vector<uint8_t> CircuitID, RemoteID;
};

class Server {
  public:
    Server(uint32_t serverIP, PoolManager *pm, ebpf::Loader *loader, Clock clock = WallClock)
        : serverIP_(serverIP), poolMgr_(pm), loader_(loader), now_(std::move(clock)) {}

    // handleDHCP, :302-383: returns the bytes to send (empty: nothing to send)
    Result<std::vector<uint8_t>> HandleDHCP(const uint8_t *pkt, size_t n) {
        Result<std::vector<uint8_t>> out;
        requestsTotal++;
        auto req = Message::Parse(pkt, n);
        if (!req.ok()) {
            out.err = req.err;
            return out;
        }
        Result<Message> resp;
        switch (req->Type()) {
        case Discover: resp = HandleDiscover(*req); break;
        case Request: resp = HandleRequest(*req); break;
        default: out.value = std::vector<uint8_t>(); return out; // RELEASE/DECLINE/INFORM: not restated
        }
        if (!resp.ok()) {
            out.err = resp.err;
            return out;
        }
        out.value = resp->ToBytes();
        return out;
    }

    Result<Message> HandleDiscover(const Message &req) { // :398-553
        Result<Message> out;
        const uint64_t mac = ebpf::MACToUint64(req.ClientHWAddr());
        uint32_t ip = 0, poolID = 0;
        std::shared_ptr<Pool> pool;
        const Lease *existing = findLease(mac);
        if (existing && now_() < existing->ExpiresAt) { // reuse the allocation of a live lease (:420-424)
            ip = existing->IP, poolID = existing->PoolID;
            pool = poolMgr_->GetPool(poolID);
        } else { // local pool (:492-508); the Nexus / HTTP-allocator branches are out of scope
            pool = poolMgr_->ClassifyClient(mac);
            if (!pool) {
                out.err = Error("no pool available for client");
                return out;
            }
            poolID = pool->ID;
            auto a = pool->Allocate(mac);
            if (!a.ok()) {
                out.err = Error("failed to allocate IP: " + a.err.what());
                return out;
            }
            ip = *a;
        }
        Message r = Message::ReplyTo(req);
        r.options[OptMessageType] = {Offer};
        r.yiaddr = ip;
        r.siaddr = serverIP_;
        r.SetIPOption(OptServerID, serverIP_);
        fillLeaseOptions(r, pool.get());
        offersTotal++;
        out.value = std::move(r);
        return out;
    }

    Result<Message> HandleRequest(const Message &req) { // :556-860, local-pool branch without RADIUS
        Result<Message> out;
        const uint64_t mac = ebpf::MACToUint64(req.ClientHWAddr());
        uint32_t requested = req.RequestedIP();
        if (!requested) requested = req.ciaddr;
        std::shared_ptr<Pool> pool;
        uint32_t poolID = 0;
        const Lease *existing = findLease(mac);
        if (existing) { // renewal: the address must match (:586-593)
            if (existing->IP != requested) return nak(req);
            pool = poolMgr_->GetPool(existing->PoolID);
            poolID = existing->PoolID;
        } else {
            pool = poolMgr_->ClassifyClient(mac);
            if (!pool) return nak(req);
            poolID = pool->ID;
            if (!pool->Contains(requested)) return nak(req);
        }
        if (!pool) return nak(req);
        Lease lease;
        lease.MAC = mac, lease.IP = requested, lease.PoolID = poolID;
        lease.ExpiresAt = now_() + pool->LeaseTimeSec;
        auto hn = req.options.find(OptHostName);
        if (hn != req.options.end()) lease.Hostname.assign(hn->second.begin(), hn->second.end());
        {
            std::lock_guard<std::mutex> g(mu_);
            leases_[mac] = lease;
        }
        fastPathError_ = updateFastPathCache(lease, *pool); // the reference logs a failure and carries on
        Message r = Message::ReplyTo(req);
        r.options[OptMessageType] = {Ack};
        r.yiaddr = requested;
        r.siaddr = serverIP_;
        r.SetIPOption(OptServerID, serverIP_);
        fillLeaseOptions(r, pool.get());
        acksTotal++;
        out.value = std::move(r);
        return out;
    }

    // seeds a lease as a previous REQUEST would have left it (test / benchmark set-up)
    void InstallLease(const Lease &l) {
        std::lock_guard<std::mutex> g(mu_);
        leases_[l.MAC] = l;
    }
    size_t ActiveLeases() {
        std::lock_guard<std::mutex> g(mu_);
        return leases_.size();
    }
    // cleanupExpiredLeases, :1115-1163, with the expired set taken from the dataplane instead of a walk over the lease
    // map: the sweep removes the expired fast-path entries of all three lease maps (the reference's RemoveSubscriber
    // leaves the VLAN and circuit-id entries behind, where they shadow a fresh lease) and reports them; each address
    // of a removed subscriber_pools entry goes back to its pool and its lease is dropped, unless it was renewed meanwhile.
    // Loops while the sweep reports more than one call returned.  Returns the entries removed, or a negative errno.
    int64_t CleanupExpiredLeases(uint64_t now_ns, const ebpf::LeaseSweepFn &sweep, uint64_t batch = 65536) {
        int64_t total = 0;
        std::vector<bng_lease_removed> recs;
        for (;;) {
            const int64_t found = sweep(now_ns, 0, batch, &recs);
            if (found < 0) return found;
            for (const auto &r : recs) {
                if (r.map != 0) continue; // a VLAN or circuit-id entry: the address stays with the subscriber's lease
                uint64_t mac;
                memcpy(&mac, r.key, 8);
                {
                    std::lock_guard<std::mutex> g(mu_);
                    auto it = leases_.find(mac);
                    if (it != leases_.end()) {
                        if ((uint64_t)it->second.ExpiresAt > r.lease_expiry) continue; // renewed since: the address is in use
                        leases_.erase(it);
                    }
                }
                // allocated_ip is the numeric value updateFastPathCache stored (BNG_LEASE_ADDR_NUMERIC)
                if (auto pool = poolMgr_->GetPool(r.pool_id)) pool->ReleaseFor(mac, r.allocated_ip);
            }
            total += (int64_t)recs.size();
            if ((uint64_t)found <= batch || recs.empty()) return total;
        }
    }
    const Error &LastFastPathError() const { return fastPathError_; }
    uint64_t requestsTotal = 0, offersTotal = 0, acksTotal = 0, naksTotal = 0;

  private:
    const Lease *findLease(uint64_t mac) {
        std::lock_guard<std::mutex> g(mu_);
        auto it = leases_.find(mac);
        return it == leases_.end() ? nullptr : &it->second;
    }
    void fillLeaseOptions(Message &r, const Pool *pool) { // :510-541: pool metadata, or 24 h and a /24 without a pool
        int64_t leaseTime = 24 * 3600;
        uint32_t mask = 0xFFFFFF00u, gateway = 0;
        std::vector<uint32_t> dns;
        if (pool) leaseTime = pool->LeaseTimeSec, mask = pool->SubnetMask, gateway = pool->Gateway, dns = pool->DNSServers;
        r.SetIPOption(OptLeaseTime, (uint32_t)leaseTime);
        r.SetIPOption(OptSubnetMask, mask);
        if (gateway) r.SetIPOption(OptRouter, gateway);
        if (!dns.empty()) {
            std::vector<uint8_t> v;
            for (uint32_t d : dns) v.insert(v.end(), {(uint8_t)(d >> 24), (uint8_t)(d >> 16), (uint8_t)(d >> 8), (uint8_t)d});
            r.options[OptDNS] = v;
        }
    }
    Result<Message> nak(const Message &req) { // buildNAK, :1043-1054
        Result<Message> out;
        naksTotal++;
        Message r = Message::ReplyTo(req);
        r.options[OptMessageType] = {Nak};
        r.siaddr = serverIP_;
        r.SetIPOption(OptServerID, serverIP_);
        out.value = std::move(r);
        return out;
    }
    Error updateFastPathCache(const Lease &lease, const Pool &pool) { // :1057-1097
        if (!loader_) return Nil();
        ebpf::PoolAssignment a;
        a.PoolID = lease.PoolID;
        a.AllocatedIP = lease.IP;
        a.VlanID = pool.VlanID;
        a.ClientClass = pool.ClientClass;
        a.LeaseExpiry = (uint64_t)lease.ExpiresAt;
        a.Flags = 0;
        Error e = loader_->AddSubscriber(lease.MAC, a);
        if (e) return e;
        if ((lease.STag > 0 || lease.CTag > 0) && loader_->HasVLANSupport()) loader_->AddVLANSubscriber(lease.STag, lease.CTag, a);
        return Nil();
    }

    uint32_t serverIP_;
    PoolManager *poolMgr_;
    ebpf::Loader *loader_;
    Clock now_;
    std::map<uint64_t, Lease> leases_;
    std::mutex mu_;
    Error fastPathError_;
};

// Pool-utilisation monitoring on the metrics ticker (FEATURES.md §9: alerts at > 80 % and > 90 % pool utilisation; the
// gauges bng_pool_utilization_ratio{pool} and bng_dhcp_active_leases of pkg/metrics).  Each Tick runs one lease census and
//   - sets Utilization(pool id, permille) for every pool ip_pools knows and ActiveLeases(unexpired subscriber_pools
//     entries);
//   - raises an alert each time a pool's permille crosses warn_permille or crit_permille upwards: once per crossing,
//     not on every tick it stays above (a fall below re-arms the level); and one per tick for a pool with conflicts.
struct PoolMonitorConfig {
    uint32_t warn_permille = 800, crit_permille = 900;
};
enum class PoolLevel { Ok = 0, Warning = 1, Critical = 2 };
struct PoolAlert {
    uint32_t PoolID = 0;
    PoolLevel Level = PoolLevel::Ok; // Ok with Conflicts > 0: an address-conflict alert
    uint32_t Permille = 0, Conflicts = 0;
};
class PoolMonitor {
  public:
    using Config = PoolMonitorConfig;
    using UtilizationFn = std::function<void(uint32_t pool_id, uint32_t permille)>;
    using ActiveLeasesFn = std::function<void(uint64_t leases)>;
    using AlertFn = std::function<void(const PoolAlert &)>;
    PoolMonitor(ebpf::LeaseCensusFn census, UtilizationFn util, ActiveLeasesFn active, AlertFn alert, Config cfg = Config())
        : census_(std::move(census)), util_(std::move(util)), active_(std::move(active)), alert_(std::move(alert)), cfg_(cfg) {}

    Result<ebpf::LeaseCensusReport> Tick(uint64_t now_ns) {
        Result<ebpf::LeaseCensusReport> r;
        ebpf::LeaseCensusReport u;
        if ((r.err = MapErr("bng_dhcp_lease_census", census_(now_ns, &u)))) return r;
        active_(u.Summary.entries[0]);
        std::map<uint32_t, PoolLevel> now;
        for (size_t i = 0; i < u.PoolIDs.size(); i++) {
            const bng_lease_pool_use &p = u.Pools[i];
            if (p.conflicts) alert_(PoolAlert{u.PoolIDs[i], PoolLevel::Ok, p.permille, p.conflicts});
            if (!p.known) continue;
            util_(u.PoolIDs[i], p.permille);
            const PoolLevel l = p.permille >= cfg_.crit_permille ? PoolLevel::Critical
                                : p.permille >= cfg_.warn_permille ? PoolLevel::Warning : PoolLevel::Ok;
            if (l == PoolLevel::Ok) continue;
            now[u.PoolIDs[i]] = l;
            if (l > Level(u.PoolIDs[i])) alert_(PoolAlert{u.PoolIDs[i], l, p.permille, p.conflicts});
        }
        level_.swap(now); // a pool missing from this census is below the warning level again
        r.value = std::move(u);
        return r;
    }
    PoolLevel Level(uint32_t pool_id) const {
        auto it = level_.find(pool_id);
        return it == level_.end() ? PoolLevel::Ok : it->second;
    }

  private:
    ebpf::LeaseCensusFn census_;
    UtilizationFn util_;
    ActiveLeasesFn active_;
    AlertFn alert_;
    Config cfg_;
    std::map<uint32_t, PoolLevel> level_;
};

// A client's DISCOVER / REQUEST as the load generator of the reference builds it (test/load/dhcp_benchmark.go:
// BOOTP payload of 300 bytes, options 53, 55 {1,3,15,6}, 255; MAC 02:00:ii:ii:ii:ii for subscriber i).
inline std::vector<uint8_t> ClientMessage(uint8_t type, uint32_t subscriber, uint32_t xid, uint32_t requestedIP = 0) {
    Message m;
    m.op = 1;
    m.xid = xid;
    m.flags = 0x8000;
    m.chaddr[0] = 0x02, m.chaddr[1] = 0x00;
    m.chaddr[2] = (uint8_t)(subscriber >> 24), m.chaddr[3] = (uint8_t)(subscriber >> 16), m.chaddr[4] = (uint8_t)(subscriber >> 8),
    m.chaddr[5] = (uint8_t)subscriber;
    m.options[OptMessageType] = {type};
    m.options[OptParamList] = {1, 3, 15, 6};
    if (requestedIP) m.SetIPOption(OptRequestedIP, requestedIP);
    return m.ToBytes();
}

} // namespace dhcp
} // namespace bng
