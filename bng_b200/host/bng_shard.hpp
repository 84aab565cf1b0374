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
//   * replication of the small read-mostly maps (ip_pools, server_config, nat_config_map, alg_ports, hairpin_ips,
//     antispoof_config, allowed_ranges_v4, nat_pool, nat_private_ranges) to every shard.
// Router::Update / Lookup / Delete are what a cgo shim binds the Go managers' Map.Put / Lookup / Delete to when
// more than one GPU is in use; Steer* is what the ingest path (RSS / flow steering) implements in hardware.
#pragma once
#include <errno.h>
#include <string.h>

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

enum class Route { ByMAC, ByPrivateIP, BySessionKey, ByEIMKey, ByReverseKey, Replicated };

inline Route RouteOf(const std::string &map) {
    if (map == "subscriber_bindings" || map == "subscriber_pools") return Route::ByMAC;
    if (map == "subscriber_nat" || map == "qos_ingress" || map == "qos_egress") return Route::ByPrivateIP;
    if (map == "nat_sessions") return Route::BySessionKey; // struct nat_key: src_ip = the subscriber's address
    if (map == "eim_table") return Route::ByEIMKey;        // struct eim_key: internal_ip
    if (map == "nat_reverse") return Route::ByReverseKey;  // struct nat_key: dst_ip/dst_port = public address, port
    return Route::Replicated;
}

// The MAC <-> IP directory and the public (address, port block) table.  Addresses are the 4 key bytes exactly as
// the maps hold them (memcpy'd into a u32), ports host order.
class Directory {
  public:
    explicit Directory(uint32_t world, uint16_t range_start = 1024, uint16_t ports_per_sub = 1024)
        : world_(world ? world : 1), range_start_(range_start), pps_(ports_per_sub ? ports_per_sub : 1024) {}
    uint32_t World() const { return world_; }
    uint32_t ShardOfMAC(uint64_t mac) const { return bng_shard_of_mac(mac, world_); }
    void Learn(uint64_t mac, uint32_t ip_key) { // lease granted: pkg/dhcp/server.go:1062-1075
        std::lock_guard<std::mutex> g(mu_);
        auto old = mac_ip_.find(mac);
        if (old != mac_ip_.end()) ip_mac_.erase(old->second);
        mac_ip_[mac] = ip_key;
        ip_mac_[ip_key] = mac;
    }
    void Forget(uint64_t mac) {
        std::lock_guard<std::mutex> g(mu_);
        auto it = mac_ip_.find(mac);
        if (it == mac_ip_.end()) return;
        ip_mac_.erase(it->second);
        mac_ip_.erase(it);
    }
    std::optional<uint32_t> ShardOfIP(uint32_t ip_key) const {
        std::lock_guard<std::mutex> g(mu_);
        auto it = ip_mac_.find(ip_key);
        if (it == ip_mac_.end()) return std::nullopt;
        return bng_shard_of_mac(it->second, world_);
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
    // ---- frame steering (what the NIC's flow steering does in front of the GPUs) ----
    static uint64_t MacKey(const uint8_t *m) {
        uint64_t k = 0;
        for (int i = 0; i < 6; i++) k = (k << 8) | m[i];
        return k;
    }
    uint32_t SteerUpstream(const uint8_t *frame, uint32_t len) const { // by source MAC
        return len >= 12 ? ShardOfMAC(MacKey(frame + 6)) : 0;
    }
    // by destination (public address, port / echo id); frames that are not translatable IPv4 go to `fallback`
    uint32_t SteerDownstream(const uint8_t *f, uint32_t len, uint32_t fallback = 0) const {
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
        if (poff + 2 > len) return fallback;
        uint16_t port = (uint16_t)((f[poff] << 8) | f[poff + 1]);
        auto s = ShardOfPublic(daddr, port);
        return s ? *s : fallback;
    }

  private:
    static constexpr uint32_t kNone = 0xFFFFFFFFu;
    uint32_t world_;
    uint16_t range_start_, pps_;
    mutable std::mutex mu_;
    std::unordered_map<uint64_t, uint32_t> mac_ip_;
    std::unordered_map<uint32_t, uint64_t> ip_mac_;
    std::unordered_map<uint32_t, std::vector<uint32_t>> blocks_; // public ip -> private ip per block index
};

// N contexts behind one map API.
class Router {
  public:
    Router(std::vector<std::shared_ptr<Backend>> shards, std::shared_ptr<Directory> dir)
        : shards_(std::move(shards)), dir_(std::move(dir)) {}
    size_t World() const { return shards_.size(); }
    Backend &Shard(size_t i) { return *shards_[i]; }
    Directory &Dir() { return *dir_; }

    // -1: replicated, -ENOENT: the owner is not known (the address was never Learn()ed)
    int Owner(const std::string &map, const void *key) const {
        const uint8_t *k = (const uint8_t *)key;
        uint32_t ip;
        switch (RouteOf(map)) {
        case Route::ByMAC: {
            uint64_t mac;
            memcpy(&mac, k, 8);
            return (int)dir_->ShardOfMAC(mac);
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
        int o = Owner(map, key);
        if (o == -ENOENT) return o;
        int rc = 0;
        for (size_t i = 0; i < shards_.size(); i++) {
            if (o >= 0 && (size_t)o != i) continue;
            bng_ctx *c = shards_[i]->ctx;
            int id = bng_map_id(c, map);
            if (id < 0) return id;
            int r = staged && flags == BNG_ANY ? bng_map_update_staged(c, id, key, value) : bng_map_update(c, id, key, value, flags);
            if (r && !rc) rc = r;
        }
        return rc;
    }
    int Lookup(const char *map, const void *key, void *value_out) {
        int o = Owner(map, key);
        if (o == -ENOENT) return o;
        bng_ctx *c = shards_[o < 0 ? 0 : (size_t)o]->ctx; // replicated maps: any copy
        int id = bng_map_id(c, map);
        return id < 0 ? id : bng_map_lookup(c, id, key, value_out);
    }
    int Delete(const char *map, const void *key) {
        int o = Owner(map, key);
        if (o == -ENOENT) return o;
        int rc = 0;
        for (size_t i = 0; i < shards_.size(); i++) {
            if (o >= 0 && (size_t)o != i) continue;
            bng_ctx *c = shards_[i]->ctx;
            int id = bng_map_id(c, map);
            if (id < 0) return id;
            int r = bng_map_delete(c, id, key);
            if (r && !rc) rc = r;
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
};

} // namespace shard
} // namespace bng
