// bng_b200 — host-side sharding of one subscriber population over N dataplane contexts (one per GPU).
//
// SURVEY.md §8(e): every mutable table is keyed by something one subscriber owns, so frames and state
// partition by  shard = splitmix64(mac_key) % N  (bng_shard_of_mac) with no data-path collective.  What the
// control plane needs on the host is
//   * the MAC <-> IP directory it already has at lease time (reference pkg/dhcp/server.go:1062-1075 hands both to
//     the fast-path cache) — per-IP maps (subscriber_nat, qos_ingress/egress, nat_sessions, eim_table) follow the
//     subscriber's MAC to its shard;
//   * for the downstream direction (§8f-1) the (public IP, port block) -> shard table.  Blocks are laid out
//     deterministically by AllocateNAT (pkg/nat/manager.go:433-434: port_start = range_start + k * ports_per_sub),
//     so the owner of an inbound (dst ip, dst port) is one array lookup;
//   * for IPv6 (subscriber_ipv6, DESIGN.md §18) the prefix -> IPv4 address table, with a longest-prefix match: a
//     prefix lives on the shard of its IPv4 address, and a downstream IPv6 frame goes to the owner of its destination;
//   * replication of the small read-mostly maps (ip_pools, server_config, nat_config_map, alg_ports, hairpin_ips,
//     antispoof_config, allowed_ranges_v4, nat_pool, nat_private_ranges) to every shard.
// Router::Update / Lookup / Delete are what a cgo shim binds the Go managers' Map.Put / Lookup / Delete to when
// more than one GPU is in use; Steer* is what the ingest path (RSS / flow steering) implements in hardware.
#pragma once
#include <errno.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/bng_b200.h"
#include "bng_host.hpp"

namespace bng {
namespace shard {

// ByValueIP: the value is the subscriber's IPv4 address (subscriber_ipv6); the entry lives on that address's shard.
// ByValueMAC: the value starts with the client's MAC (dhcpv6_bindings); the entry lives on that MAC's shard, where the
// client's upstream frames are steered.
enum class Route { ByMAC, ByPrivateIP, BySessionKey, ByEIMKey, ByReverseKey, ByValueIP, ByValueMAC, Replicated };

inline Route RouteOf(const std::string &map) {
    if (map == "subscriber_bindings" || map == "subscriber_pools" || map == "nd_bindings") return Route::ByMAC;
    if (map == "subscriber_nat" || map == "qos_ingress" || map == "qos_egress") return Route::ByPrivateIP;
    if (map == "nat_sessions") return Route::BySessionKey; // struct nat_key: src_ip = the subscriber's address
    if (map == "eim_table") return Route::ByEIMKey;        // struct eim_key: internal_ip
    if (map == "nat_reverse") return Route::ByReverseKey;  // struct nat_key: dst_ip/dst_port = public address, port
    if (map == "subscriber_ipv6") return Route::ByValueIP; // value: the owner's IPv4 address
    if (map == "dhcpv6_bindings") return Route::ByValueMAC; // value: struct bng_dhcpv6_binding, mac first
    return Route::Replicated;
}

// The MAC <-> IP directory and the public (address, port block) table.  Addresses are the 4 key bytes exactly as
// the maps hold them (memcpy'd into a u32), ports host order.
class Directory {
  public:
    explicit Directory(uint32_t world, uint16_t range_start = 1024, uint16_t ports_per_sub = 1024)
        : world_(world ? world : 1), range_start_(range_start), pps_(ports_per_sub ? ports_per_sub : 1024) {}
    uint32_t World() const { return world_; }
    // The owner of a MAC: its pin (Router::Move), else bng_shard_of_mac.  Every other route derives from this one.
    uint32_t ShardOfMAC(uint64_t mac) const {
        std::lock_guard<std::mutex> g(mu_);
        return ShardOfMACLocked(mac);
    }
    // A pin overrides the hash for one MAC: a subscriber whose state was moved to another shard stays there.  It lasts
    // until Unpin or Forget.
    void Pin(uint64_t mac, uint32_t shard) {
        std::lock_guard<std::mutex> g(mu_);
        pins_[mac] = shard;
    }
    void Unpin(uint64_t mac) {
        std::lock_guard<std::mutex> g(mu_);
        pins_.erase(mac);
    }
    // (MAC, address) of every learned subscriber whose owner is shard k
    std::vector<std::pair<uint64_t, uint32_t>> SubscribersOn(uint32_t k) const {
        std::lock_guard<std::mutex> g(mu_);
        std::vector<std::pair<uint64_t, uint32_t>> out;
        for (const auto &e : mac_ip_)
            if (ShardOfMACLocked(e.first) == k) out.push_back(e);
        std::sort(out.begin(), out.end());
        return out;
    }
    void Learn(uint64_t mac, uint32_t ip_key) { // lease granted: pkg/dhcp/server.go:1062-1075
        std::lock_guard<std::mutex> g(mu_);
        auto old = mac_ip_.find(mac);
        if (old != mac_ip_.end()) ip_mac_.erase(old->second);
        mac_ip_[mac] = ip_key;
        ip_mac_[ip_key] = mac;
    }
    // The subscriber is gone: its address mapping (unless the address has been learned for another MAC since) and its
    // pin go with it, so a returning MAC is placed by bng_shard_of_mac again.
    void Forget(uint64_t mac) {
        std::lock_guard<std::mutex> g(mu_);
        pins_.erase(mac);
        auto it = mac_ip_.find(mac);
        if (it == mac_ip_.end()) return;
        auto ip = ip_mac_.find(it->second);
        if (ip != ip_mac_.end() && ip->second == mac) ip_mac_.erase(ip);
        mac_ip_.erase(it);
    }
    std::optional<uint32_t> ShardOfIP(uint32_t ip_key) const {
        std::lock_guard<std::mutex> g(mu_);
        auto it = ip_mac_.find(ip_key);
        if (it == ip_mac_.end()) return std::nullopt;
        return ShardOfMACLocked(it->second);
    }
    // AllocateNAT gave `private_ip_key` the block [port_start, port_end] of public_ip_key
    void AddBlock(uint32_t public_ip_key, uint16_t port_start, uint32_t private_ip_key) {
        std::lock_guard<std::mutex> g(mu_);
        auto &v = blocks_[public_ip_key];
        size_t k = (size_t)(port_start - range_start_) / pps_;
        if (v.size() <= k) v.resize(k + 1, kNone);
        v[k] = private_ip_key;
    }
    void RemoveBlock(uint32_t public_ip_key, uint16_t port_start) {
        std::lock_guard<std::mutex> g(mu_);
        auto it = blocks_.find(public_ip_key);
        if (it == blocks_.end()) return;
        size_t k = (size_t)(port_start - range_start_) / pps_;
        if (k < it->second.size()) it->second[k] = kNone;
    }
    // owner of an inbound frame addressed to (public ip, port): the subscriber holding that block
    std::optional<uint32_t> ShardOfPublic(uint32_t public_ip_key, uint16_t port) const {
        uint32_t priv;
        {
            std::lock_guard<std::mutex> g(mu_);
            auto it = blocks_.find(public_ip_key);
            if (it == blocks_.end() || port < range_start_) return std::nullopt;
            size_t k = (size_t)(port - range_start_) / pps_;
            if (k >= it->second.size() || it->second[k] == kNone) return std::nullopt;
            priv = it->second[k];
        }
        return ShardOfIP(priv);
    }
    // ---- IPv6 prefixes (subscriber_ipv6): prefix -> IPv4 address key, longest-prefix match ----
    using Addr6 = std::array<uint8_t, 16>;
    static Addr6 Masked(const uint8_t *addr, uint32_t plen) {
        Addr6 a;
        for (uint32_t j = 0; j < 16; j++) {
            const uint32_t keep = plen >= 8 * (j + 1) ? 8 : (plen > 8 * j ? plen - 8 * j : 0);
            a[j] = (uint8_t)(addr[j] & (uint8_t)(0xFF00u >> keep));
        }
        return a;
    }
    // false for prefixlen > 128
    bool LearnPrefix(const uint8_t *addr, uint32_t plen, uint32_t ip_key) {
        if (plen > 128) return false;
        std::lock_guard<std::mutex> g(mu_);
        v6_[plen][Masked(addr, plen)] = ip_key;
        return true;
    }
    void ForgetPrefix(const uint8_t *addr, uint32_t plen) {
        if (plen > 128) return;
        std::lock_guard<std::mutex> g(mu_);
        v6_[plen].erase(Masked(addr, plen));
    }
    // the IPv4 address of exactly this prefix
    std::optional<uint32_t> PrefixOwner(const uint8_t *addr, uint32_t plen) const {
        if (plen > 128) return std::nullopt;
        std::lock_guard<std::mutex> g(mu_);
        auto it = v6_[plen].find(Masked(addr, plen));
        if (it == v6_[plen].end()) return std::nullopt;
        return it->second;
    }
    // the IPv4 address of the longest prefix of length <= maxlen covering addr (the dataplane's rule)
    std::optional<uint32_t> OwnerOfV6(const uint8_t *addr, uint32_t maxlen = 128) const {
        std::lock_guard<std::mutex> g(mu_);
        for (int l = (int)std::min<uint32_t>(maxlen, 128); l >= 0; l--) {
            if (v6_[l].empty()) continue;
            auto it = v6_[l].find(Masked(addr, (uint32_t)l));
            if (it != v6_[l].end()) return it->second;
        }
        return std::nullopt;
    }
    std::optional<uint32_t> ShardOfV6(const uint8_t *addr) const {
        auto ip = OwnerOfV6(addr);
        return ip ? ShardOfIP(*ip) : std::nullopt;
    }
    // ---- frame steering (what the NIC's flow steering does in front of the GPUs) ----
    static uint64_t MacKey(const uint8_t *m) {
        uint64_t k = 0;
        for (int i = 0; i < 6; i++) k = (k << 8) | m[i];
        return k;
    }
    uint32_t SteerUpstream(const uint8_t *frame, uint32_t len) const { // by source MAC
        return len >= 12 ? ShardOfMAC(MacKey(frame + 6)) : 0;
    }
    // IPv4: by destination (public address, port / echo id).  IPv6 (untagged, ethertype 0x86DD): by the owner of the
    // longest prefix covering the destination (bytes 38-53), the shard that holds its records.  Anything else, and a
    // destination nobody owns, goes to `fallback`.  With ICMP error translation on (SetICMPErrors), an ICMP error
    // (type 3, 11 or 12) goes by the flow it quotes: (quoted source, quoted source port or ICMP id), when the frame is
    // one nat44_ingress can translate; otherwise to `fallback`, since every shard passes it unchanged.
    uint32_t SteerDownstream(const uint8_t *f, uint32_t len, uint32_t fallback = 0) const {
        if (len >= 54 && f[12] == 0x86 && f[13] == 0xDD) {
            auto s = ShardOfV6(f + 38);
            return s ? *s : fallback;
        }
        if (len < 34 || f[12] != 0x08 || f[13] != 0x00) return fallback;
        uint32_t l4 = 14 + (uint32_t)(f[14] & 0x0f) * 4, daddr;
        memcpy(&daddr, f + 30, 4);
        uint32_t proto = f[23], poff;
        if (proto == 6 || proto == 17)
            poff = l4 + 2;
        else if (proto == 1)
            poff = l4 + 4;
        else
            return fallback;
        if (proto == 1 && icmp_errors_.load(std::memory_order_relaxed) && l4 + 8 <= len &&
            (f[l4] == 3 || f[l4] == 11 || f[l4] == 12)) {
            // the length first: a quoted byte is read only once the frame holds it (66: the TCP/UDP ports, the least a
            // translatable error carries)
            if (l4 != 34 || len < 66) return fallback;
            const uint32_t ip = f[51];
            if (f[42] != 0x45 || (ip != 6 && ip != 17 && ip != 1) || memcmp(f + 54, f + 30, 4)) return fallback;
            const uint32_t qoff = ip == 1 ? 66 : 62; // the quoted ICMP id / source port: the public port
            if (ip == 1 && len < 68) return fallback;
            uint32_t qsrc;
            memcpy(&qsrc, f + 54, 4);
            auto s = ShardOfPublic(qsrc, (uint16_t)((f[qoff] << 8) | f[qoff + 1]));
            return s ? *s : fallback;
        }
        if (poff + 2 > len) return fallback;
        uint16_t port = (uint16_t)((f[poff] << 8) | f[poff + 1]);
        auto s = ShardOfPublic(daddr, port);
        return s ? *s : fallback;
    }

    // SteerDownstream keys ICMP errors by the flow they quote (Router::NatICMPErrorsEnable)
    void SetICMPErrors(bool on) { icmp_errors_.store(on, std::memory_order_relaxed); }

  private:
    uint32_t ShardOfMACLocked(uint64_t mac) const {
        if (!pins_.empty()) {
            auto p = pins_.find(mac);
            if (p != pins_.end()) return p->second;
        }
        return bng_shard_of_mac(mac, world_);
    }
    static constexpr uint32_t kNone = 0xFFFFFFFFu;
    uint32_t world_;
    std::unordered_map<uint64_t, uint32_t> pins_; // MAC -> shard, set by Router::Move
    uint16_t range_start_, pps_;
    std::atomic<bool> icmp_errors_{false};
    mutable std::mutex mu_;
    std::unordered_map<uint64_t, uint32_t> mac_ip_;
    std::unordered_map<uint32_t, uint64_t> ip_mac_;
    std::unordered_map<uint32_t, std::vector<uint32_t>> blocks_; // public ip -> private ip per block index
    std::array<std::map<Addr6, uint32_t>, 129> v6_;               // per prefix length: masked prefix -> IPv4 key
};

// N contexts behind one map API.
class Router {
  public:
    Router(std::vector<std::shared_ptr<Backend>> shards, std::shared_ptr<Directory> dir)
        : shards_(std::move(shards)), dir_(std::move(dir)) {}
    size_t World() const { return shards_.size(); }
    Backend &Shard(size_t i) { return *shards_[i]; }
    Directory &Dir() { return *dir_; }

    // -1: replicated, -ENOENT: the owner is not known (the address was never Learn()ed).  subscriber_ipv6 (ByValueIP):
    // with the value, the owner of its IPv4 address; without it, the owner of the prefix as the directory learned it.
    int Owner(const std::string &map, const void *key, const void *value = nullptr) const {
        const uint8_t *k = (const uint8_t *)key;
        uint32_t ip;
        switch (RouteOf(map)) {
        case Route::ByValueIP: {
            uint32_t plen;
            memcpy(&plen, k, 4);
            if (plen > 128) return -EINVAL;
            std::optional<uint32_t> a;
            if (value) {
                memcpy(&ip, value, 4);
                a = ip;
            } else {
                a = dir_->PrefixOwner(k + 4, plen);
            }
            if (!a) return -ENOENT;
            auto s = dir_->ShardOfIP(*a);
            return s ? (int)*s : -ENOENT;
        }
        case Route::ByMAC: {
            uint64_t mac;
            memcpy(&mac, k, 8);
            return (int)dir_->ShardOfMAC(mac);
        }
        case Route::ByValueMAC: { // with the value, the shard of its MAC; without it, the shard that holds the key
            if (value) return (int)dir_->ShardOfMAC(Directory::MacKey((const uint8_t *)value));
            std::lock_guard<std::mutex> g(home_mu_);
            auto it = home_.find(std::string((const char *)key, 32));
            return it == home_.end() ? -ENOENT : (int)it->second;
        }
        case Route::ByPrivateIP:
        case Route::BySessionKey:
        case Route::ByEIMKey: {
            memcpy(&ip, k, 4);
            auto s = dir_->ShardOfIP(ip);
            return s ? (int)*s : -ENOENT;
        }
        case Route::ByReverseKey: {
            memcpy(&ip, k + 4, 4); // nat_key.dst_ip = the public address
            uint16_t port = (uint16_t)((k[10] << 8) | k[11]);
            auto s = dir_->ShardOfPublic(ip, port);
            return s ? (int)*s : -ENOENT;
        }
        default: return -1;
        }
    }
    int Update(const char *map, const void *key, const void *value, uint64_t flags = BNG_ANY, bool staged = false) {
        const bool v6 = RouteOf(map) == Route::ByValueIP;
        int o = Owner(map, key, value);
        if (o == -ENOENT || o == -EINVAL) return o;
        if (v6) { // a prefix handed to another subscriber leaves its old shard
            const int was = Owner(map, key);
            if (was >= 0 && was != o) {
                bng_ctx *c = shards_[(size_t)was]->ctx;
                const int id = bng_map_id(c, map);
                if (id < 0) return id;
                if (int r = bng_map_delete(c, id, key); r && r != -ENOENT) return r;
            }
        }
        if (RouteOf(map) == Route::ByValueMAC) { // a client re-bound under another MAC leaves its old shard
            const int was = Owner(map, key);
            if (was >= 0 && was != o) {
                bng_ctx *c = shards_[(size_t)was]->ctx;
                const int id = bng_map_id(c, map);
                if (id < 0) return id;
                if (int r = bng_map_delete(c, id, key); r && r != -ENOENT) return r;
                std::lock_guard<std::mutex> g(home_mu_);
                home_.erase(std::string((const char *)key, 32));
            }
        }
        int rc = 0;
        for (size_t i = 0; i < shards_.size(); i++) {
            if (o >= 0 && (size_t)o != i) continue;
            bng_ctx *c = shards_[i]->ctx;
            int id = bng_map_id(c, map);
            if (id < 0) return id;
            int r = staged && flags == BNG_ANY ? bng_map_update_staged(c, id, key, value) : bng_map_update(c, id, key, value, flags);
            if (r && !rc) rc = r;
        }
        if (RouteOf(map) == Route::ByValueMAC && !rc) {
            std::lock_guard<std::mutex> g(home_mu_);
            home_[std::string((const char *)key, 32)] = (size_t)o;
        }
        if (v6 && !rc) {
            uint32_t plen, a;
            memcpy(&plen, key, 4);
            memcpy(&a, value, 4);
            dir_->LearnPrefix((const uint8_t *)key + 4, plen, a);
        }
        return rc;
    }
    int Lookup(const char *map, const void *key, void *value_out) {
        int o;
        if (RouteOf(map) == Route::ByValueIP) { // the longest match: its owner's shard answers
            uint32_t plen;
            memcpy(&plen, key, 4);
            if (plen > 128) return -EINVAL;
            auto a = dir_->OwnerOfV6((const uint8_t *)key + 4, plen);
            auto s = a ? dir_->ShardOfIP(*a) : std::nullopt;
            if (!s) return -ENOENT;
            o = (int)*s;
        } else {
            o = Owner(map, key);
        }
        if (o == -ENOENT) return o;
        bng_ctx *c = shards_[o < 0 ? 0 : (size_t)o]->ctx; // replicated maps: any copy
        int id = bng_map_id(c, map);
        return id < 0 ? id : bng_map_lookup(c, id, key, value_out);
    }
    int Delete(const char *map, const void *key) {
        int o = Owner(map, key);
        if (o == -ENOENT || o == -EINVAL) return o;
        if (RouteOf(map) == Route::ByValueIP) {
            uint32_t plen;
            memcpy(&plen, key, 4);
            dir_->ForgetPrefix((const uint8_t *)key + 4, plen);
        }
        int rc = 0;
        for (size_t i = 0; i < shards_.size(); i++) {
            if (o >= 0 && (size_t)o != i) continue;
            bng_ctx *c = shards_[i]->ctx;
            int id = bng_map_id(c, map);
            if (id < 0) return id;
            int r = bng_map_delete(c, id, key);
            if (r && !rc) rc = r;
        }
        if (RouteOf(map) == Route::ByValueMAC && (!rc || rc == -ENOENT)) {
            std::lock_guard<std::mutex> g(home_mu_);
            home_.erase(std::string((const char *)key, 32));
        }
        return rc;
    }
    // Per-subscriber traffic record (bng_acct_read) from the shard that owns the address: upstream frames follow
    // the subscriber's MAC to it and downstream frames are steered to it by (public address, port block)
    // (SteerDownstream), so its record is the whole record and no other shard holds one.
    int AcctOwner(uint32_t addr_key) const {
        auto s = dir_->ShardOfIP(addr_key);
        return s ? (int)*s : -ENOENT;
    }
    int AcctRead(uint32_t addr_key, bng_acct *out) {
        int o = AcctOwner(addr_key);
        if (o < 0) return o;
        int32_t res = 0;
        int rc = bng_acct_read(shards_[(size_t)o]->ctx, &addr_key, 1, out, &res);
        return rc ? rc : res;
    }
    // NAT flow-state flush (bng_nat_flush) of addresses given as subscriber_nat key words.  A subscriber's sessions,
    // reverse entries and EIM mappings are all created on its owner shard (downstream frames are steered there by
    // public address and port block), so each address goes to its owner; one whose owner is not known goes to every
    // shard, where a flush of an address without state is a no-op.  One call per shard that has addresses.
    // removed_out (may be null): sessions, reverse entries, EIM mappings removed, summed over the shards.
    std::vector<std::vector<uint32_t>> NatFlushGroups(const uint32_t *addrs, uint64_t n) const {
        std::vector<std::vector<uint32_t>> g(shards_.size());
        for (uint64_t i = 0; i < n; i++) {
            auto s = dir_->ShardOfIP(addrs[i]);
            for (size_t k = 0; k < shards_.size(); k++)
                if (!s || *s == k) g[k].push_back(addrs[i]);
        }
        return g;
    }
    int NatFlush(const uint32_t *addrs, uint64_t n, uint64_t now_ns, uint64_t removed_out[3] = nullptr) {
        if (removed_out) removed_out[0] = removed_out[1] = removed_out[2] = 0;
        if (n && !addrs) return -EINVAL;
        auto g = NatFlushGroups(addrs, n);
        int rc = 0;
        for (size_t k = 0; k < g.size(); k++) {
            if (g[k].empty()) continue;
            uint64_t rm[3] = {0, 0, 0};
            int r = bng_nat_flush(shards_[k]->ctx, g[k].data(), g[k].size(), now_ns, rm);
            if (r && !rc) rc = r;
            if (removed_out)
                for (int j = 0; j < 3; j++) removed_out[j] += rm[j];
        }
        return rc;
    }
    // Lawful-intercept targets (bng_li_target_set / _del) go to the shard that owns the address: its upstream frames
    // follow the subscriber's MAC there, and downstream frames are steered there by (public address, port block).  An
    // address whose owner is not known goes to every shard.  Del returns -ENOENT when no shard had the target.
    std::vector<size_t> LiShards(uint32_t addr_key) const {
        auto s = dir_->ShardOfIP(addr_key);
        std::vector<size_t> out;
        for (size_t k = 0; k < shards_.size(); k++)
            if (!s || *s == k) out.push_back(k);
        return out;
    }
    int LiTargetSet(uint32_t addr_key, uint32_t target_id) {
        for (size_t k : LiShards(addr_key))
            if (int r = bng_li_target_set(shards_[k]->ctx, addr_key, target_id)) return r;
        return 0;
    }
    int LiTargetDel(uint32_t addr_key) {
        int rc = -ENOENT;
        for (size_t k : LiShards(addr_key)) {
            int r = bng_li_target_del(shards_[k]->ctx, addr_key);
            if (r == 0) rc = 0;
            else if (r != -ENOENT) return r;
        }
        return rc;
    }
    // IPv6 shaping (bng_qos_ipv6_enable) on every shard: one bucket per subscriber whatever the address family.  A
    // subscriber's IPv6 frames already reach its shard (SteerDownstream, and upstream by MAC), so each shard shapes
    // them with the bucket it holds.  Returns 0 or the first shard's error.
    int QoSIPv6Enable(bool on) {
        for (auto &s : shards_)
            if (int r = bng_qos_ipv6_enable(s->ctx, on ? 1 : 0)) return r;
        return 0;
    }
    // Antispoof by delegated prefix (bng_antispoof_ipv6_prefixes_enable) on every shard.  The rule needs a
    // subscriber's binding and its prefixes on one shard: the binding is routed ByMAC and subscriber_ipv6 ByValueIP,
    // the shard of the IPv4 address and so of its MAC.  Returns 0 or the first shard's error.
    // The DHCPv6 fast path (bng_dhcpv6_enable) on every shard.  dhcpv6_bindings is routed ByValueMAC and
    // dhcpv6_server_config replicated, and upstream frames are steered by source MAC (SteerUpstream), so a client's
    // messages reach the shard that holds its binding.  Returns 0 or the first shard's error.
    int DHCPv6Enable(bool on) {
        for (auto &s : shards_)
            if (int r = bng_dhcpv6_enable(s->ctx, on ? 1 : 0)) return r;
        return 0;
    }
    int AntispoofIPv6PrefixesEnable(bool on) {
        for (auto &s : shards_)
            if (int r = bng_antispoof_ipv6_prefixes_enable(s->ctx, on ? 1 : 0)) return r;
        return 0;
    }
    // Router and Neighbor Solicitations answered on the GPU (bng_nd_enable) on every shard.  nd_bindings is routed ByMAC
    // and nd_config replicated, and upstream frames are steered by source MAC, so a subscriber's RS reaches the shard
    // that holds its binding.  Returns 0 or the first shard's error.
    int NDEnable(bool on) {
        for (auto &s : shards_)
            if (int r = bng_nd_enable(s->ctx, on ? 1 : 0)) return r;
        return 0;
    }
    // ICMP error translation in nat44_ingress (bng_nat_icmp_errors_enable) on every shard, and SteerDownstream sends an
    // ICMP error to the shard of the flow it quotes (without it, the error's bytes 4-5 name no block and it goes to
    // `fallback`, which holds no session).  Returns 0 or the first shard's error.
    int NatICMPErrorsEnable(bool on) {
        for (auto &s : shards_)
            if (int r = bng_nat_icmp_errors_enable(s->ctx, on ? 1 : 0)) return r;
        dir_->SetICMPErrors(on);
        return 0;
    }
    // Upstream ICMP error translation (bng_nat_icmp_errors_egress_enable) on every shard.  No steering change:
    // SteerUpstream goes by source MAC, so a subscriber's error reaches its own shard, which holds the quoted session.
    // Returns 0 or the first shard's error.
    int NatICMPErrorsEgressEnable(bool on) {
        for (auto &s : shards_)
            if (int r = bng_nat_icmp_errors_egress_enable(s->ctx, on ? 1 : 0)) return r;
        return 0;
    }
    // Drains every shard: fn(shard, record, record size) per record, in (batch, frame) order within a shard (batch
    // numbers are per shard).  Returns the number of records or a negative errno.
    template <class F>
    int64_t LiDrain(F &&fn, uint64_t batch = 4096) {
        int64_t total = 0;
        for (size_t k = 0; k < shards_.size(); k++) {
            const uint32_t rs = bng_li_record_size(shards_[k]->ctx);
            if (!rs) continue;
            std::vector<uint8_t> buf((size_t)batch * rs);
            for (;;) {
                uint64_t n = 0;
                if (int r = bng_li_drain(shards_[k]->ctx, buf.data(), batch, &n)) return r;
                for (uint64_t i = 0; i < n; i++) fn(k, buf.data() + i * rs, rs);
                total += (int64_t)n;
                if (n < batch) break;
            }
        }
        return total;
    }
    // Incremental replication: shard k of the active node replicates to shard k of the standby node (the same
    // subscribers steer to the same shard index on both), so each pair is independent and no collective is needed.
    // DeltaExport writes shard k's delta into *out; DeltaApply applies, on shard k of the standby, the delta its peer
    // exported.  Both return 0 or a negative errno (-ESTALE: the pair needs a FULL delta).
    int DeltaExport(size_t k, uint64_t refresh_ns, uint32_t flags, std::vector<uint8_t> *out) {
        if (k >= shards_.size() || !out) return -EINVAL;
        out->resize(std::max<size_t>(out->capacity(), 1 << 16));
        for (;;) {
            uint64_t len = 0;
            int r = bng_delta_export(shards_[k]->ctx, refresh_ns, flags, out->data(), out->size(), &len);
            if (r == -ENOSPC && len > out->size()) {
                out->resize(len);
                continue;
            }
            out->resize(r ? 0 : len);
            return r;
        }
    }
    int DeltaApply(size_t k, const void *blob, uint64_t len) {
        if (k >= shards_.size()) return -EINVAL;
        return bng_delta_apply(shards_[k]->ctx, blob, len);
    }
    // Subscriber hand-over (bng_sub_export / bng_sub_import): the state of `addrs` (subscriber_nat key words) and
    // `macs` leaves shard `from` and is taken by shard `to`; on success the MACs are pinned to `to`, so every route
    // (ShardOfMAC, ShardOfIP, ShardOfPublic, Steer*, Owner and the per-address calls above) follows them there.
    // When `to` refuses the blob, it goes back into `from` (the import restores a context exactly), the pins stay as
    // they were and the import's error is returned.  Should `from` refuse it too, the state is on neither shard:
    // Move returns -ENOTRECOVERABLE and hands the blob to `stranded` (when given) for a later bng_sub_import.  The
    // blob passes through host memory.
    int Move(size_t from, size_t to, const std::vector<uint32_t> &addrs, const std::vector<uint64_t> &macs,
             std::vector<uint8_t> *stranded = nullptr) {
        if (from >= shards_.size() || to >= shards_.size() || from == to) return -EINVAL;
        std::vector<uint8_t> blob(1 << 16);
        for (;;) {
            uint64_t len = 0;
            int r = bng_sub_export(shards_[from]->ctx, addrs.data(), addrs.size(), macs.data(), macs.size(), BNG_SUB_DETACH,
                                   blob.data(), blob.size(), &len);
            if (r == -ENOSPC && len > blob.size()) {
                blob.resize(len);
                continue;
            }
            if (r) return r;
            blob.resize(len);
            break;
        }
        int r = bng_sub_import(shards_[to]->ctx, blob.data(), blob.size());
        if (r) {
            if (bng_sub_import(shards_[from]->ctx, blob.data(), blob.size()) == 0) return r;
            if (stranded) *stranded = std::move(blob);
            return -ENOTRECOVERABLE;
        }
        for (uint64_t m : macs) dir_->Pin(m, (uint32_t)to);
        return 0;
    }
    // Destination of a subscriber drained off shard k: the bng_shard_of_mac(mac, N - 1)-th of the other shards.
    size_t DrainTarget(size_t k, uint64_t mac) const {
        const size_t j = bng_shard_of_mac(mac, (uint32_t)shards_.size() - 1);
        return j < k ? j : j + 1;
    }
    // Takes shard k out of service: every subscriber the directory places there moves, MAC and address, to
    // DrainTarget; one Move per destination.  Returns 0 or the first error (the subscribers of the destinations
    // before it have moved).
    int Drain(size_t k) {
        if (k >= shards_.size() || shards_.size() < 2) return -EINVAL;
        std::vector<std::vector<uint32_t>> a(shards_.size());
        std::vector<std::vector<uint64_t>> m(shards_.size());
        for (const auto &e : dir_->SubscribersOn((uint32_t)k)) {
            const size_t t = DrainTarget(k, e.first);
            m[t].push_back(e.first);
            a[t].push_back(e.second);
        }
        for (size_t t = 0; t < shards_.size(); t++)
            if (!m[t].empty())
                if (int r = Move(k, t, a[t], m[t])) return r;
        return 0;
    }
    // Idle detection (bng_idle_*).  A subscriber's record lives on its owner shard only: upstream frames follow its MAC
    // there and downstream frames are steered there by (public address, port block), so the owner's record is the
    // whole record and no collective is needed.  IdleTimeoutSet sends each address to its owner, or to every shard
    // when the owner is not known; results[i] is 0 when some shard had an entry for it, else -ENOENT.
    int IdleTimeoutSet(const uint32_t *addrs, const uint32_t *timeouts_s, uint64_t n, int32_t *results) {
        if (n && (!addrs || !timeouts_s || !results)) return -EINVAL;
        std::vector<std::vector<uint64_t>> idx(shards_.size());
        for (uint64_t i = 0; i < n; i++) {
            results[i] = -ENOENT;
            for (size_t k : LiShards(addrs[i])) idx[k].push_back(i);
        }
        for (size_t k = 0; k < shards_.size(); k++) {
            if (idx[k].empty()) continue;
            std::vector<uint32_t> a, t;
            for (uint64_t i : idx[k]) a.push_back(addrs[i]), t.push_back(timeouts_s[i]);
            std::vector<int32_t> res(a.size());
            if (int r = bng_idle_timeout_set(shards_[k]->ctx, a.data(), t.data(), a.size(), res.data())) return r;
            for (size_t j = 0; j < a.size(); j++)
                if (res[j] == 0) results[idx[k][j]] = 0;
        }
        return 0;
    }
    // Every shard's scan: returns the idle records found over all shards and writes the first cap of them.
    int64_t IdleScan(uint64_t now_ns, uint32_t default_s, uint32_t flags, uint32_t *addrs_out, bng_idle *out, uint64_t cap) {
        if (cap && (!addrs_out || !out)) return -EINVAL;
        int64_t total = 0;
        for (auto &s : shards_) {
            const uint64_t at = std::min<uint64_t>((uint64_t)total, cap);
            int64_t n = bng_idle_scan(s->ctx, now_ns, default_s, flags, cap > at ? addrs_out + at : nullptr,
                                      cap > at ? out + at : nullptr, cap - at);
            if (n < 0) return n;
            total += n;
        }
        return total;
    }
    // Records of n addresses, each from its owner (or, when the owner is not known, from the shard that has it).
    int IdleRead(const uint32_t *addrs, uint64_t n, bng_idle *out, int32_t *results) {
        if (n && (!addrs || !out || !results)) return -EINVAL;
        for (uint64_t i = 0; i < n; i++) {
            out[i] = bng_idle{};
            results[i] = -ENOENT;
            for (size_t k : LiShards(addrs[i])) {
                bng_idle rec{};
                int32_t res = 0;
                if (int r = bng_idle_read(shards_[k]->ctx, &addrs[i], 1, &rec, &res)) return r;
                if (res == 0) {
                    out[i] = rec, results[i] = 0;
                    break;
                }
            }
        }
        return 0;
    }
    // NAT port-usage census (bng_nat_usage) over every shard.  Each shard counts its own tables: a subscriber's record
    // comes from the shard that holds its subscriber_nat entry (its owner), public-address records are merged by address
    // with every field summed, and the summaries are summed.  A triple held on two shards (overlapping blocks, DESIGN.md
    // §8) counts once per shard.
    int NatUsage(uint32_t min_permille, nat::PortUsageReport *out) {
        if (!out) return -EINVAL;
        std::vector<nat::PortUsageReport> parts(shards_.size());
        for (size_t k = 0; k < shards_.size(); k++)
            if (int r = nat::ContextPortUsage(shards_[k]->ctx, min_permille, &parts[k])) return r;
        *out = MergeNatUsage(parts);
        return 0;
    }
    static nat::PortUsageReport MergeNatUsage(const std::vector<nat::PortUsageReport> &parts) {
        nat::PortUsageReport m;
        std::map<uint32_t, bng_nat_pub_use> pubs;
        for (const auto &p : parts) {
            const uint64_t *a = (const uint64_t *)&p.Summary;
            uint64_t *s = (uint64_t *)&m.Summary;
            for (size_t i = 0; i < sizeof(bng_nat_usage_sum) / 8; i++) s[i] += a[i];
            m.SubAddrs.insert(m.SubAddrs.end(), p.SubAddrs.begin(), p.SubAddrs.end());
            m.Subs.insert(m.Subs.end(), p.Subs.begin(), p.Subs.end());
            for (size_t i = 0; i < p.PubAddrs.size(); i++) {
                auto ins = pubs.emplace(p.PubAddrs[i], p.Pubs[i]);
                if (ins.second) continue;
                bng_nat_pub_use &t = ins.first->second;
                const bng_nat_pub_use &u = p.Pubs[i];
                t.sessions += u.sessions, t.eim += u.eim, t.block_ports += u.block_ports, t.blocks += u.blocks;
                for (int c = 0; c < 3; c++) t.in_use[c] += u.in_use[c];
                t.in_use_any += u.in_use_any, t.unreachable += u.unreachable;
            }
        }
        for (auto &kv : pubs) m.PubAddrs.push_back(kv.first), m.Pubs.push_back(kv.second);
        m.Summary.pubs_found = pubs.size();
        return m;
    }
    // DHCP lease census over every shard.  Each shard counts its own tables: pool records are merged by pool_id with the
    // counts summed (prefix_hosts and known taken from any shard that has them, permille recomputed), and the summaries
    // are summed.  An address leased on two shards counts once per shard in addrs, and a conflict between two shards'
    // subscribers is not seen: subscribers are sharded by MAC, so a pool's addresses are spread over the shards.
    int LeaseCensus(uint64_t now_ns, ebpf::LeaseCensusReport *out) {
        if (!out) return -EINVAL;
        std::vector<ebpf::LeaseCensusReport> parts(shards_.size());
        for (size_t k = 0; k < shards_.size(); k++)
            if (int r = ebpf::ContextLeaseCensus(shards_[k]->ctx, now_ns, &parts[k])) return r;
        *out = MergeLeaseCensus(parts);
        return 0;
    }
    static ebpf::LeaseCensusReport MergeLeaseCensus(const std::vector<ebpf::LeaseCensusReport> &parts) {
        ebpf::LeaseCensusReport m;
        std::map<uint32_t, bng_lease_pool_use> pools;
        for (const auto &p : parts) {
            const uint64_t *a = (const uint64_t *)&p.Summary;
            uint64_t *s = (uint64_t *)&m.Summary;
            for (size_t i = 0; i < sizeof(bng_lease_sum) / 8; i++) s[i] += a[i];
            for (size_t i = 0; i < p.PoolIDs.size(); i++) {
                auto ins = pools.emplace(p.PoolIDs[i], p.Pools[i]);
                if (ins.second) continue;
                bng_lease_pool_use &t = ins.first->second;
                const bng_lease_pool_use &u = p.Pools[i];
                for (int c = 0; c < 3; c++) t.entries[c] += u.entries[c];
                t.expired += u.expired, t.addrs += u.addrs, t.addrs_outside += u.addrs_outside, t.conflicts += u.conflicts;
                if (u.known) t.known = 1, t.prefix_hosts = u.prefix_hosts;
            }
        }
        for (auto &kv : pools) {
            bng_lease_pool_use &t = kv.second;
            t.permille = t.prefix_hosts ? (uint32_t)((uint64_t)(t.addrs - t.addrs_outside) * 1000 / t.prefix_hosts) : 0;
            m.PoolIDs.push_back(kv.first), m.Pools.push_back(t);
        }
        m.Summary.pools_found = pools.size();
        return m;
    }
    // Every shard's sweep, concatenated: at most `cap` entries removed per shard; returns the due entries found over
    // all shards (repeat while it exceeds what came back).
    int64_t LeaseSweep(uint64_t now_ns, uint32_t grace_s, uint64_t cap, std::vector<bng_lease_removed> *out) {
        if (!out) return -EINVAL;
        out->clear();
        int64_t total = 0;
        std::vector<bng_lease_removed> part;
        for (auto &s : shards_) {
            int64_t n = ebpf::ContextLeaseSweep(s->ctx, now_ns, grace_s, cap, &part);
            if (n < 0) return n;
            total += n;
            out->insert(out->end(), part.begin(), part.end());
        }
        return total;
    }
    nat::UsageFn NatUsageSource() {
        return [this](uint32_t min_permille, nat::PortUsageReport *out) { return NatUsage(min_permille, out); };
    }
    idle::TimeoutSetFn IdleTimeoutSetter() {
        return [this](const uint32_t *a, const uint32_t *t, uint64_t n, int32_t *res) { return IdleTimeoutSet(a, t, n, res); };
    }
    idle::ScanFn IdleScanner() {
        return [this](uint64_t now, uint32_t def, uint32_t flags, uint32_t *a, bng_idle *o, uint64_t cap) {
            return IdleScan(now, def, flags, a, o, cap);
        };
    }
    radius::AcctReader Reader() {
        return [this](uint32_t addr, bng_acct *out) { return AcctRead(addr, out); };
    }
    // PERCPU-style totals: the packed counter vector summed over the shards (host-side sum; with a communicator
    // per context bng_sync_reduce() does the same on the devices)
    int Totals(uint64_t out[BNG_NUM_STATS]) {
        memset(out, 0, sizeof(uint64_t) * BNG_NUM_STATS);
        for (auto &s : shards_) {
            uint64_t v[BNG_NUM_STATS];
            int r = bng_sync_reduce(s->ctx, v);
            if (r) return r;
            for (int i = 0; i < BNG_NUM_STATS; i++) out[i] += v[i];
        }
        return 0;
    }

  private:
    std::vector<std::shared_ptr<Backend>> shards_;
    std::shared_ptr<Directory> dir_;
    // dhcpv6_bindings (ByValueMAC): the shard that holds each key, so that delete and lookup find it and a re-bind
    // under another MAC can leave the old shard
    mutable std::mutex home_mu_;
    std::unordered_map<std::string, size_t> home_;
};

} // namespace shard
} // namespace bng
