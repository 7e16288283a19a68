// gpu_object_placement.hpp -- C++ mirror of the reference's provider interface over the C ABI (include/rio_cuda.h).
//
//   trait ObjectPlacement { prepare, update, lookup, clean_server, remove }   rio-rs/src/object_placement/mod.rs:38-56
//   ObjectPlacementItem { object_id, server_address: Option<String> }         rio-rs/src/object_placement/mod.rs:20-34
//   ObjectId(String, String)                                                  rio-rs/src/service_object.rs:19-26
//   ObjectPlacementError::{Upstream, Unknown}                                 rio-rs/src/errors.rs:136-142
//
// Same names, argument meaning and error behaviour as the Rust trait (Result<T, E> becomes a thrown
// ObjectPlacementError; Option<String> becomes std::optional<std::string>).  Header-only; link with -lrio_cuda.
#pragma once
#include <cstdint>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../include/rio_cuda.h"

namespace rio_rs {

struct ObjectId {                      // service_object.rs:19-26
    std::string struct_name, object_id;
    ObjectId(std::string t, std::string i) : struct_name(std::move(t)), object_id(std::move(i)) {}
};

struct ObjectPlacementItem {           // mod.rs:20-34
    ObjectId object_id;
    std::optional<std::string> server_address;
    ObjectPlacementItem(ObjectId id, std::optional<std::string> addr) : object_id(std::move(id)), server_address(std::move(addr)) {}
};

struct ObjectPlacementError : std::runtime_error {   // errors.rs:136-142
    enum Kind { Upstream, Unknown } kind;
    ObjectPlacementError(Kind k, const std::string &m) : std::runtime_error(m), kind(k) {}
};

class GpuObjectPlacement {
    struct Engine {
        rio_placement *h = nullptr;
        ~Engine() { if (h) rio_cuda_destroy(h); }
    };
    std::shared_ptr<Engine> e_;        // Clone shares state (local.rs:12-18)

    void check(rio_status st) const {
        if (st == RIO_OK) return;
        const char *m = rio_cuda_last_error(e_ ? e_->h : nullptr);
        throw ObjectPlacementError(st == RIO_ERR_UPSTREAM ? ObjectPlacementError::Upstream : ObjectPlacementError::Unknown, m ? m : "");
    }

  public:
    explicit GpuObjectPlacement(int device = -1, uint64_t directory_capacity = 0) : e_(std::make_shared<Engine>()) {
        rio_config cfg{(uint32_t)sizeof(rio_config), device, directory_capacity, 0, 0};
        rio_status st = rio_cuda_create(&cfg, &e_->h);
        if (st != RIO_OK) {
            const char *m = rio_cuda_last_error(nullptr);
            throw ObjectPlacementError(st == RIO_ERR_UPSTREAM ? ObjectPlacementError::Upstream : ObjectPlacementError::Unknown, m ? m : "");
        }
    }
    GpuObjectPlacement clone() const { return *this; }
    rio_placement *handle() const { return e_->h; }

    // ---- the trait ------------------------------------------------------------------------------------------
    void prepare() const {}                                                             // mod.rs:41-43
    void update(const ObjectPlacementItem &it) const {                                  // mod.rs:46-49
        const std::string &t = it.object_id.struct_name, &i = it.object_id.object_id;
        check(rio_cuda_update_str(e_->h, t.data(), t.size(), i.data(), i.size(), it.server_address ? it.server_address->data() : nullptr,
                                  it.server_address ? it.server_address->size() : 0));
    }
    std::optional<std::string> lookup(const ObjectId &id) const {                       // mod.rs:51
        std::string buf(256, '\0');
        for (;;) {   // the call reports the full length; an address longer than the buffer is read again into one that fits
            size_t len = 0;
            check(rio_cuda_lookup_str(e_->h, id.struct_name.data(), id.struct_name.size(), id.object_id.data(), id.object_id.size(), &buf[0], buf.size(), &len));
            if (len == (size_t)-1) return std::nullopt;
            if (len <= buf.size()) { buf.resize(len); return buf; }
            buf.assign(len, '\0');
        }
    }
    void clean_server(const std::string &address) const { check(rio_cuda_clean_server_str(e_->h, address.data(), address.size())); }   // mod.rs:53
    void remove(const ObjectId &id) const {                                             // mod.rs:55
        check(rio_cuda_remove_str(e_->h, id.struct_name.data(), id.struct_name.size(), id.object_id.data(), id.object_id.size()));
    }

    // ---- batched extensions -----------------------------------------------------------------------------------
    static uint64_t object_key(const ObjectId &id) {
        return rio_cuda_object_key(id.struct_name.data(), id.struct_name.size(), id.object_id.data(), id.object_id.size());
    }
    std::vector<uint32_t> set_nodes(const std::vector<std::string> &addrs, const std::vector<uint32_t> *weights = nullptr) const {
        std::vector<const char *> p;
        for (auto &a : addrs) p.push_back(a.c_str());
        std::vector<uint32_t> out(addrs.size());
        check(rio_cuda_set_nodes(e_->h, p.data(), weights ? weights->data() : nullptr, nullptr, (uint32_t)addrs.size(), 0, out.data()));
        return out;
    }
    void node_set_active(uint32_t idx, bool active) const { check(rio_cuda_node_set_active(e_->h, idx, active)); }
    // failure-domain labels (DESIGN.md 3.12): a rack or zone id per node, RIO_NONE = a domain of its own
    void set_node_domains(const std::vector<uint32_t> &idx, const std::vector<uint32_t> &domain) const {
        if (idx.size() != domain.size()) throw ObjectPlacementError(ObjectPlacementError::Unknown, "idx and domain differ in length");
        check(rio_cuda_node_set_domains(e_->h, idx.data(), domain.data(), idx.size()));
    }
    uint32_t node_domain(uint32_t idx) const { uint32_t d = RIO_NONE; check(rio_cuda_node_domain(e_->h, idx, &d)); return d; }
    std::string node_address(uint32_t idx) const {
        size_t len = 0;
        check(rio_cuda_node_address(e_->h, idx, nullptr, 0, &len));      // the length first, then the bytes
        std::string a(len, '\0');
        if (len) check(rio_cuda_node_address(e_->h, idx, &a[0], a.size(), &len));
        return a;
    }
    std::vector<uint32_t> lookup_many(const std::vector<uint64_t> &keys) const {
        std::vector<uint32_t> out(keys.size());
        check(rio_cuda_lookup_batch(e_->h, keys.data(), keys.size(), out.data()));
        return out;
    }
    void update_many(const std::vector<uint64_t> &keys, const std::vector<uint32_t> &idx) const {
        check(rio_cuda_upsert_batch(e_->h, keys.data(), idx.data(), keys.size()));
    }
    std::vector<uint32_t> assign_batch(const std::vector<uint64_t> &keys) const {
        std::vector<uint32_t> out(keys.size());
        check(rio_cuda_assign_batch(e_->h, keys.data(), nullptr, keys.size(), out.data()));
        return out;
    }
    // each object's first `ranks` distinct nodes (DESIGN.md 3.9), row-major: object i's list at [i * ranks, (i + 1) * ranks)
    std::vector<uint32_t> assign_ranked(const std::vector<uint64_t> &keys, uint32_t ranks) const {
        std::vector<uint32_t> out(keys.size() * ranks);
        check(rio_cuda_assign_ranked_batch(e_->h, keys.data(), keys.size(), ranks, out.data()));
        return out;
    }
    // each object's first `ranks` nodes in distinct failure domains (DESIGN.md 3.12), row-major as for assign_ranked
    std::vector<uint32_t> assign_ranked_spread(const std::vector<uint64_t> &keys, uint32_t ranks) const {
        std::vector<uint32_t> out(keys.size() * ranks);
        check(rio_cuda_assign_ranked_spread_batch(e_->h, keys.data(), keys.size(), ranks, out.data()));
        return out;
    }
    // each object's `ranks` lowest-cost live nodes under the affinity cost (DESIGN.md 3.9); obj_feats is n x K row-major (K of
    // set_nodes), the result row-major as for assign_ranked
    std::vector<uint32_t> assign_ranked_affinity(const std::vector<float> &obj_feats, size_t n, uint32_t ranks) const {
        if (n && obj_feats.size() % n) throw ObjectPlacementError(ObjectPlacementError::Unknown, "obj_feats is not n x K");
        std::vector<uint32_t> out(n * ranks);
        check(rio_cuda_assign_ranked_affinity_batch(e_->h, obj_feats.data(), n, ranks, out.data()));
        return out;
    }
    // each object's `ranks` lowest-cost live nodes in distinct failure domains under the affinity cost (DESIGN.md 3.14), arguments
    // and result as for assign_ranked_affinity
    std::vector<uint32_t> assign_ranked_affinity_spread(const std::vector<float> &obj_feats, size_t n, uint32_t ranks) const {
        if (n && obj_feats.size() % n) throw ObjectPlacementError(ObjectPlacementError::Unknown, "obj_feats is not n x K");
        std::vector<uint32_t> out(n * ranks);
        check(rio_cuda_assign_ranked_affinity_spread_batch(e_->h, obj_feats.data(), n, ranks, out.data()));
        return out;
    }
    std::vector<uint32_t> place_batch(const std::vector<uint64_t> &keys, uint32_t policy, uint32_t self_idx) const {
        std::vector<uint32_t> out(keys.size());
        check(rio_cuda_place_batch(e_->h, keys.data(), keys.size(), policy, self_idx, out.data()));
        return out;
    }
    uint64_t rebalance(uint32_t event, uint32_t idx) const { uint64_t m = 0; check(rio_cuda_rebalance(e_->h, event, idx, &m)); return m; }
    // one pass for a set of node changes (DESIGN.md 3.10): {node index, its weight before the change if it was live then, else 0}
    uint64_t rebalance_changes(const std::vector<std::pair<uint32_t, uint32_t>> &changes) const {
        std::vector<uint32_t> idx, prev;
        for (const auto &c : changes) { idx.push_back(c.first); prev.push_back(c.second); }
        uint64_t m = 0;
        check(rio_cuda_rebalance_changes(e_->h, idx.data(), prev.data(), idx.size(), &m));
        return m;
    }
};

}  // namespace rio_rs
