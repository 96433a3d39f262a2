// slot_cache.hpp -- residency of tenants in a fixed set of device regions: which tenant holds which region, and which region a
// batch's missing tenants take.  Pure host bookkeeping (no device call); B200Server's key pager (key-bank slots, assignAll) and c1
// store (cached c1 rows, assignByCount) issue the fills it decides.
#pragma once
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

namespace evab {

class RegionCache {
public:
  struct Fill { int tenant, region, evicted; };   // evicted: the tenant the region held before, -1 if it was free

  explicit RegionCache(int regions) : owner_(regions, -1), stamp_(regions, 0) {
    if (regions < 1) throw std::invalid_argument("a region cache needs at least one region");
  }
  int regions() const { return (int)owner_.size(); }
  int regionOf(int tenant) const { auto it = region_.find(tenant); return it == region_.end() ? -1 : it->second; }
  // tenants holding a region, in region order
  std::vector<int> holders() const {
    std::vector<int> r;
    for (int t : owner_) if (t >= 0) r.push_back(t);
    return r;
  }
  std::uint64_t fills() const { return fills_; }
  std::uint64_t evictions() const { return evictions_; }

  // Key-bank slots: the slot of every instance of a batch.  Every distinct tenant of the batch is pinned: the tenants already
  // resident keep their slots, and each missing one (in order of first appearance) takes the lowest free slot, else the least
  // recently used slot that no tenant of this batch holds.  Each distinct tenant is stamped in that order.  `fills` receives the
  // slots to fill.  More distinct tenants than slots is an error, raised before anything changes.
  std::vector<int> assignAll(const std::vector<int> &tenants, std::vector<Fill> &fills) {
    std::vector<int> distinct;
    for (int t : tenants)
      if (std::find(distinct.begin(), distinct.end(), t) == distinct.end()) distinct.push_back(t);
    if ((int)distinct.size() > regions())
      throw std::invalid_argument("a batch names " + std::to_string(distinct.size()) + " distinct tenants but the key bank has " +
                                  std::to_string(regions()) + " device slots");
    std::vector<char> pinned = pin(distinct);
    for (int t : distinct) {
      int s = regionOf(t);
      if (s < 0) s = take(t, pinned, fills);
      stamp_[s] = ++clock_;
    }
    std::vector<int> out;
    out.reserve(tenants.size());
    for (int t : tenants) out.push_back(region_.at(t));
    return out;
  }
  // Cached c1 rows: the region of every instance of a batch, -1: the instance draws.  Unlike bank slots, a batch may name more
  // distinct tenants than there are regions.  Admission order: the tenants with more instances in the batch first, ties by first
  // appearance; the first regions() of them are admitted.  Admitted tenants that hold a region keep it (pinned); each missing one,
  // in admission order, takes the lowest free region, else the least recently used region that no admitted tenant holds.  `fills`
  // receives the regions to fill.  Every instance whose tenant then holds a region reads it -- a tenant left out of admission keeps
  // its region while no admitted tenant needs it -- and the batch stamps those regions once.
  std::vector<int> assignByCount(const std::vector<int> &tenants, std::vector<Fill> &fills) {
    std::vector<int> order;           // distinct tenants by first appearance
    std::unordered_map<int, int> count;
    for (int t : tenants)
      if (count[t]++ == 0) order.push_back(t);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return count[a] > count[b]; });
    if ((int)order.size() > regions()) order.resize(regions());
    std::vector<char> pinned = pin(order);
    for (int t : order)
      if (regionOf(t) < 0) take(t, pinned, fills);
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
  // the regions the admitted tenants already hold
  std::vector<char> pin(const std::vector<int> &admitted) const {
    std::vector<char> pinned(regions(), 0);
    for (int t : admitted) if (int r = regionOf(t); r >= 0) pinned[r] = 1;
    return pinned;
  }
  // a missing admitted tenant takes the victim region, which it pins
  int take(int tenant, std::vector<char> &pinned, std::vector<Fill> &fills) {
    const int r = victim(pinned);
    const int old = owner_[r];
    if (old >= 0) { region_.erase(old); evictions_++; }
    owner_[r] = tenant; region_[tenant] = r; pinned[r] = 1;
    fills.push_back(Fill{tenant, r, old});
    fills_++;
    return r;
  }
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
