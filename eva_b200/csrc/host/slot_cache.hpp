// slot_cache.hpp -- residency of key-bank tenants in device slots: which tenant holds which slot, and which slot a batch's missing
// tenants take.  Pure host bookkeeping (no device call); B200Server's key pager issues the fills it decides.
#pragma once
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

namespace evab {

class SlotCache {
public:
  struct Fill { int tenant, slot, evicted; };   // evicted: the tenant the slot held before, -1 if it was free

  explicit SlotCache(int slots) : owner_(slots, -1), stamp_(slots, 0) {
    if (slots < 1) throw std::invalid_argument("a slot cache needs at least one slot");
  }
  int slots() const { return (int)owner_.size(); }
  int slotOf(int tenant) const { auto it = slot_.find(tenant); return it == slot_.end() ? -1 : it->second; }
  // tenants holding a slot, in slot order
  std::vector<int> resident() const {
    std::vector<int> r;
    for (int t : owner_) if (t >= 0) r.push_back(t);
    return r;
  }
  std::uint64_t fills() const { return fills_; }
  std::uint64_t evictions() const { return evictions_; }

  // The slot of every instance of a batch.  Every distinct tenant of the batch is pinned: the tenants already resident keep their
  // slots, and each missing one (in order of first appearance) takes the lowest free slot, else the least recently used slot
  // that no tenant of this batch holds.  `fills` receives the slots to fill.  More distinct tenants than slots is an error, raised
  // before anything changes.
  std::vector<int> assign(const std::vector<int> &tenants, std::vector<Fill> &fills) {
    std::vector<int> distinct;
    for (int t : tenants)
      if (std::find(distinct.begin(), distinct.end(), t) == distinct.end()) distinct.push_back(t);
    if ((int)distinct.size() > slots())
      throw std::invalid_argument("a batch names " + std::to_string(distinct.size()) + " distinct tenants but the key bank has " +
                                  std::to_string(slots()) + " device slots");
    std::vector<char> pinned(slots(), 0);
    for (int t : distinct) if (int s = slotOf(t); s >= 0) pinned[s] = 1;
    for (int t : distinct) {
      int s = slotOf(t);
      if (s < 0) {
        s = victim(pinned);
        const int old = owner_[s];
        if (old >= 0) { slot_.erase(old); evictions_++; }
        owner_[s] = t; slot_[t] = s; pinned[s] = 1;
        fills.push_back(Fill{t, s, old});
        fills_++;
      }
      stamp_[s] = ++clock_;
    }
    std::vector<int> out;
    out.reserve(tenants.size());
    for (int t : tenants) out.push_back(slot_.at(t));
    return out;
  }
  // the tenant's keys are gone: its slot (if any) becomes free
  void drop(int tenant) {
    auto it = slot_.find(tenant);
    if (it == slot_.end()) return;
    owner_[it->second] = -1; stamp_[it->second] = 0;
    slot_.erase(it);
  }

private:
  int victim(const std::vector<char> &pinned) const {
    for (int s = 0; s < slots(); s++) if (owner_[s] < 0) return s;
    int best = -1;
    for (int s = 0; s < slots(); s++)
      if (!pinned[s] && (best < 0 || stamp_[s] < stamp_[best])) best = s;
    return best;   // exists: the batch pins at most slots() - 1 slots while one of its tenants is missing
  }
  std::vector<int> owner_;                 // slot -> tenant, -1: free
  std::vector<std::uint64_t> stamp_;       // slot -> last batch use (LRU)
  std::unordered_map<int, int> slot_;      // tenant -> slot
  std::uint64_t clock_ = 0, fills_ = 0, evictions_ = 0;
};

// Residency of tenants' cached c1 rows (B200Server c1_cache): which tenant holds which of a seeded bank's c1 regions, and which
// regions a batch's tenants take.  Unlike bank slots, a batch may name more distinct tenants than there are regions: the tenants
// left out draw their c1 rows in the kernels, as without a cache.
class C1Cache {
public:
  struct Fill { int tenant, region, evicted; };   // evicted: the tenant the region held before, -1 if it was free

  explicit C1Cache(int regions) : owner_(regions, -1), stamp_(regions, 0) {
    if (regions < 1) throw std::invalid_argument("a c1 cache needs at least one region");
  }
  int regions() const { return (int)owner_.size(); }
  int regionOf(int tenant) const { auto it = region_.find(tenant); return it == region_.end() ? -1 : it->second; }
  // tenants holding a region, in region order
  std::vector<int> cached() const {
    std::vector<int> r;
    for (int t : owner_) if (t >= 0) r.push_back(t);
    return r;
  }
  std::uint64_t fills() const { return fills_; }
  std::uint64_t evictions() const { return evictions_; }

  // The region of every instance of a batch, -1: the instance draws.  Admission order: the tenants with more instances in the batch
  // first, ties by first appearance; the first regions() of them are admitted.  Admitted tenants that hold a region keep it
  // (pinned); each missing one, in admission order, takes the lowest free region, else the least recently used region that no
  // admitted tenant holds.  `fills` receives the regions to fill.  Every instance whose tenant then holds a region reads it -- a
  // tenant left out of admission keeps its region while no admitted tenant needs it.
  std::vector<int> assign(const std::vector<int> &tenants, std::vector<Fill> &fills) {
    std::vector<int> order;           // distinct tenants by first appearance
    std::unordered_map<int, int> count;
    for (int t : tenants)
      if (count[t]++ == 0) order.push_back(t);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return count[a] > count[b]; });
    if ((int)order.size() > regions()) order.resize(regions());
    std::vector<char> pinned(regions(), 0);
    for (int t : order) if (int r = regionOf(t); r >= 0) pinned[r] = 1;
    for (int t : order) {
      if (regionOf(t) >= 0) continue;
      const int r = victim(pinned);
      const int old = owner_[r];
      if (old >= 0) { region_.erase(old); evictions_++; }
      owner_[r] = t; region_[t] = r; pinned[r] = 1;
      fills.push_back(Fill{t, r, old});
      fills_++;
    }
    ++clock_;
    std::vector<int> out;
    out.reserve(tenants.size());
    for (int t : tenants) {
      const int r = regionOf(t);
      if (r >= 0) stamp_[r] = clock_;
      out.push_back(r);
    }
    return out;
  }
  // the tenant's keys are gone: its region (if any) becomes free
  void drop(int tenant) {
    auto it = region_.find(tenant);
    if (it == region_.end()) return;
    owner_[it->second] = -1; stamp_[it->second] = 0;
    region_.erase(it);
  }

private:
  int victim(const std::vector<char> &pinned) const {
    for (int r = 0; r < regions(); r++) if (owner_[r] < 0) return r;
    int best = -1;
    for (int r = 0; r < regions(); r++)
      if (!pinned[r] && (best < 0 || stamp_[r] < stamp_[best])) best = r;
    return best;   // exists: at most regions() tenants are admitted, and one of them is missing
  }
  std::vector<int> owner_;                 // region -> tenant, -1: free
  std::vector<std::uint64_t> stamp_;       // region -> last batch use (LRU)
  std::unordered_map<int, int> region_;    // tenant -> region
  std::uint64_t clock_ = 0, fills_ = 0, evictions_ = 0;
};

}  // namespace evab
