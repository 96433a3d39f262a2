// backend.hpp -- the GPU counterpart of the reference's SEAL backend API
// (eva/seal/seal.h:24-97, eva/seal/seal.cpp): generateKeys, B200Public::{encrypt,
// execute}, B200Secret::decrypt, B200Valuation.  Same argument meaning, ownership
// and error behaviour (C++ exceptions -> Python exceptions through pybind11).
#pragma once
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include "executor.hpp"
#include "slot_cache.hpp"
#include <atomic>
#include <functional>
#include <mutex>
#include <tuple>
#include <variant>

namespace evab {

// compiler outputs (reference eva/ckks/ckks_parameters.h:14-18, ckks_signature.h:16-36)
struct CKKSParameters {
  std::vector<std::uint32_t> primeBits;
  std::set<int> rotations;
  std::uint32_t polyModulusDegree = 0;
};
struct CKKSEncodingInfo {
  Type inputType; int scale; int level;
  CKKSEncodingInfo(Type t, int s, int l) : inputType(t), scale(s), level(l) {}
};
struct CKKSSignature {
  int vecSize = 0;
  std::map<std::string, CKKSEncodingInfo> inputs;
  CKKSSignature() {}
  CKKSSignature(int v, std::map<std::string, CKKSEncodingInfo> in) : vecSize(v), inputs(std::move(in)) {}
};
using Valuation = std::map<std::string, std::vector<double>>;

// The rotation steps that get a Galois key.  "program": every step of the program (the compiler's rotation set, step 0 included).
// "power_of_two": the distinct NAF terms of its nonzero steps but those of magnitude N/2, ascending; every rotation of the program
// is then composed from them as SEAL's rotate_vector does (planner.hpp composeRotations)
inline std::vector<int> rotationKeySteps(const CKKSParameters &params, const std::string &rotationKeys) {
  if (rotationKeys == "program") return std::vector<int>(params.rotations.begin(), params.rotations.end());
  if (rotationKeys != "power_of_two") throw std::invalid_argument("rotation_keys must be \"program\" or \"power_of_two\", not \"" + rotationKeys + "\"");
  std::set<int> steps;
  for (int s : params.rotations) {
    if (!s) continue;
    if (!evab_host::galois_elt_from_step(params.polyModulusDegree, s)) throw std::invalid_argument("step count too large");
    for (int t : evab_host::naf_rotation_terms(params.polyModulusDegree, s)) steps.insert(t);
  }
  return std::vector<int>(steps.begin(), steps.end());
}

// host-resident encrypted values (the reference keeps seal::Ciphertext objects
// in host memory inside SEALValuation, eva/seal/seal.h:21-41)
// host images of ciphertexts / plaintexts live in page-locked memory (asynchronous, full-rate H2D / D2H)
struct HostCipher { HostBuf data; int size = 0, ell = 0; double scale = 0; };
struct HostPlain { HostBuf data; int ell = 0; double scale = 0; };
// a seed-compressed fresh ciphertext (B200Secret::encrypt): c0 [ell][N] and the seed of c1 (key_expand.cuh, ciphertext rows);
// always size 2.  A type of its own, so that no reader of HostCipher can take its ell N words for 2 ell N
struct HostSeededCipher { HostBuf c0; int ell = 0; double scale = 0; KeySeed seed{}; };
// a reference to a ciphertext held in a B200Server's store (CipherStore): the handle alone; level, scale and words are the entry's
struct StoredCipher { std::uint64_t handle = 0; };
// a compact response (B200Public compact_outputs): an output ciphertext switched to the modulus 2^bits and bit-packed,
// words [2][W], W = ceil(N bits / 64) (compact_kernels.cuh); scale is the compact scale.  Decrypted by B200Secret, never a program input
struct HostCompactCipher { HostBuf words; int bits = 0; double scale = 0; };
using SchemeValue = std::variant<HostCipher, HostPlain, std::shared_ptr<ConstantValue>, HostSeededCipher, StoredCipher, HostCompactCipher>;

// Compact responses: the modulus 2^bits an output ciphertext at `ell` residues, scale `scale` and declared range `range` (bits) is
// switched to for `precision` bits after the binary point, with margin m = log2 N + 1 for the rounding noise r0 + r1 s.
//   shift = ceil(log2(Q / scale)) + precision + m,  bits = min(shift, range + precision + m + 2),  compact scale = scale 2^shift / Q
// (log2 Q is the sum of log2 q_i).  The whole policy: the output stays a full ciphertext when it is not a ciphertext, has size 3,
// declares no range (no width can be derived), has more than kCompactMaxEll residues (the CRT limit of the compaction kernel),
// bits >= floor(log2 Q) (nothing would shrink) or bits > 62.  Decided on the host before anything of a batch is enqueued
constexpr int kCompactMaxEll = 8;   // evab_compact_ciphers / evab_compact_finish / evab_decode residue limit
struct CompactShape { bool compact = false; int shift = 0, bits = 0; double scale = 0; };
inline CompactShape compactShape(const std::vector<u64> &primes, bool cipher, int size, int ell, double scale, std::optional<std::uint32_t> range,
                                 int precision, u64 N) {
  CompactShape c;
  if (!cipher || size != 2 || !range || ell < 1 || ell > (int)primes.size()) return c;
  double log2Q = 0;
  for (int i = 0; i < ell; i++) log2Q += std::log2((double)primes[i]);
  const int m = (int)std::log2((double)N) + 1;
  c.shift = (int)std::ceil(log2Q - std::log2(scale)) + precision + m;
  c.bits = std::min(c.shift, (int)*range + precision + m + 2);
  c.scale = std::pow(2.0, std::log2(scale) + c.shift - log2Q);
  c.compact = c.bits < (int)std::floor(log2Q) && c.bits <= 62 && ell <= kCompactMaxEll;
  return c;
}
// the one refusal of a compact value where a ciphertext is expected
inline std::invalid_argument compactRefused(const std::string &what) {
  return std::invalid_argument(what + " is a compact response (compact_outputs): it can only be decrypted, not sent to a program or stored");
}

class B200Valuation {
public:
  SchemeValue &operator[](const std::string &name) { return values[name]; }
  const SchemeValue &at(const std::string &name) const { return values.at(name); }
  auto begin() const { return values.begin(); }
  auto end() const { return values.end(); }
  std::size_t size() const { return values.size(); }
  std::map<std::string, SchemeValue> values;
};

// Ordering of device regions that a fill stream rewrites while runs on other streams read them: a fill waits for the runs that
// may still read its region (one reader event per region and reader stream), and records the region's fill event, which every run
// that reads the region waits for.  The host never blocks on the way.
class RegionFences {
public:
  RegionFences(std::shared_ptr<Device> dev, int regions) : dev_(std::move(dev)), fillEv_(regions, nullptr), readers_(regions) {
    check(evab_stream_create(dev_->ctx(), &stream_));
  }
  ~RegionFences() {
    evab_ctx *c = dev_->ctx();
    evab_sync(c, stream_);
    for (void *e : fillEv_) if (e) evab_event_destroy(c, e);
    for (auto &m : readers_) for (auto &r : m) evab_event_destroy(c, r.second);
    evab_stream_destroy(c, stream_);
  }
  RegionFences(const RegionFences &) = delete;
  // the fill stream
  void *stream() const { return stream_; }
  // the fill stream waits for every run recorded as a reader of region r
  void awaitReaders(int r) {
    for (auto &e : readers_[r]) check(evab_stream_wait_event(dev_->ctx(), stream_, e.second));
  }
  // a fill of region r has been enqueued on the fill stream
  void filled(int r) {
    if (!fillEv_[r]) check(evab_event_create(dev_->ctx(), &fillEv_[r]));
    check(evab_event_record(dev_->ctx(), fillEv_[r], stream_));
  }
  // the event of the last fill of region r (null: never filled)
  void *fillEvent(int r) const { return fillEv_[r]; }
  // a run on `stream` that reads the regions of `entries` (entry e >= 0: region e - base; e < 0: none) waits for their fills; once
  // enqueued, it is recorded as their reader on that stream
  void beforeRun(void *stream, const int *entries, int n, int base = 0) {
    for (int i = 0; i < n; i++)
      if (firstOf(entries, i))
        if (void *ev = fillEv_[entries[i] - base]) check(evab_stream_wait_event(dev_->ctx(), stream, ev));
  }
  void afterRun(void *stream, const int *entries, int n, int base = 0) {
    for (int i = 0; i < n; i++) {
      if (!firstOf(entries, i)) continue;
      void *&ev = readers_[entries[i] - base][stream];
      if (!ev) check(evab_event_create(dev_->ctx(), &ev));
      check(evab_event_record(dev_->ctx(), ev, stream));
    }
  }

private:
  // entries[i] names a region that entries[0 .. i) does not
  static bool firstOf(const int *entries, int i) { return entries[i] >= 0 && std::find(entries, entries + i, entries[i]) == entries + i; }
  std::shared_ptr<Device> dev_;
  std::vector<void *> fillEv_;                      // region -> event of its last fill
  std::vector<std::map<void *, void *>> readers_;   // region -> (reader stream -> event after its last run that read the region)
  void *stream_ = nullptr;                          // fills
};

// Paging of evaluation keys (B200Server with more tenants than key-bank regions): every registered tenant's keys live in a
// page-locked host block (in full, or compressed: c0 rows and seeds, expanded on the device at every fill), and the bank's regions
// are device slots holding the keys of the tenants used recently (RegionCache::assignAll).  A batch's missing tenants are filled on
// the pager's fill stream, ordered against the runs by the slots' RegionFences: a fill uploads the keys and recomputes the slot's
// hoist constants.
class KeyPager {
public:
  KeyPager(std::shared_ptr<Device> dev, KeyBank &bank, int maxTenants)
      : dev_(std::move(dev)), bank_(bank), cache_(bank.capacity()), host_(maxTenants), fences_(dev_, bank.capacity()) {}
  ~KeyPager() {
    evab_sync(dev_->ctx(), fences_.stream());   // fills still reading the host blocks (fences_ is destroyed after this body)
    for (Block &h : host_) if (h.p) evab_host_free(h.p);
  }
  int maxTenants() const { return (int)host_.size(); }
  int tenants() const { return (int)std::count_if(host_.begin(), host_.end(), [](const Block &h) { return h.p != nullptr; }); }
  int compressedTenants() const { return (int)std::count_if(host_.begin(), host_.end(), [](const Block &h) { return h.p && h.compressed; }); }
  bool registered(int t) const { return t >= 0 && t < maxTenants() && host_[t].p; }
  void requireRegistered(int t) const {
    if (!registered(t)) throw std::invalid_argument("tenant " + std::to_string(t) + " has no keys on this server");
  }
  // host images [k-1][2][k][N] of the relinearization key and of every element's Galois key (checked by the caller) into a new
  // page-locked block; no device work.  Returns the tenant id
  int add(const u64 *relinKey, const std::map<u64, const u64 *> &galoisKeys) {
    if (bank_.seededKeys()) throw std::logic_error("a bank of seeded keys takes compressed keys only");
    Block &b = freeBlock(bank_.keyWords(), false);
    const std::size_t kw = bank_.keyWords() / bank_.keys();
    std::memcpy(b.p, relinKey, kw * 8);
    for (std::size_t i = 0; i < bank_.elements().size(); i++) std::memcpy(b.p + kw * (1 + i), galoisKeys.at(bank_.elements()[i]), kw * 8);
    return (int)(&b - host_.data());
  }
  // a compressed tenant: c0 rows and seeds (KeyBank::packCompressed), half the bytes of a full one
  int addCompressed(const u64 *relinC0, const KeySeed &relinSeed, const std::map<u64, std::pair<const u64 *, KeySeed>> &galois) {
    Block &b = freeBlock(bank_.compressedWords(), true);
    bank_.packCompressed(b.p, relinC0, relinSeed, galois);
    return (int)(&b - host_.data());
  }
  void remove(int t) {
    requireRegistered(t);
    cache_.drop(t);
    check(evab_sync(dev_->ctx(), fences_.stream()));   // a fill may still be reading the block
    evab_host_free(host_[t].p);
    host_[t] = Block();
  }
  // the slot of every instance of a batch; the missing tenants' fills are enqueued on the pager's stream
  std::vector<int> resolve(const std::vector<int> &tenants) {
    std::vector<RegionCache::Fill> fills;
    std::vector<int> slots = cache_.assignAll(tenants, fills);
    for (auto &f : fills) {
      fences_.awaitReaders(f.region);
      const Block &b = host_[f.tenant];
      if (b.compressed) bank_.fillCompressed(f.region, b.p, fences_.stream());
      else bank_.fill(f.region, b.p, fences_.stream());
      fences_.filled(f.region);
    }
    return slots;
  }
  // a run on `stream` that reads `slots` waits for their fills; once enqueued, it is recorded as their reader on that stream
  void beforeRun(void *stream, const int *slots, int n) { fences_.beforeRun(stream, slots, n); }
  void afterRun(void *stream, const int *slots, int n) { fences_.afterRun(stream, slots, n); }
  const RegionCache &cache() const { return cache_; }
  // the event of the last fill of a slot (null: never filled by the pager)
  void *fillEvent(int slot) const { return fences_.fillEvent(slot); }
  std::size_t hostBytes() const {
    std::size_t w = 0;
    for (const Block &b : host_) w += b.words;
    return w * 8;
  }

private:
  struct Block {
    u64 *p = nullptr;          // page-locked; null: free id
    std::size_t words = 0;     // KeyBank::keyWords() (full) or compressedWords()
    bool compressed = false;
  };
  Block &freeBlock(std::size_t words, bool compressed) {
    const auto it = std::find_if(host_.begin(), host_.end(), [](const Block &h) { return h.p == nullptr; });
    if (it == host_.end()) throw std::runtime_error("the host key store is full (" + std::to_string(maxTenants()) + " tenants): remove a tenant first");
    check(evab_host_alloc(words * 8, (void **)&it->p));
    it->words = words; it->compressed = compressed;
    return *it;
  }
  std::shared_ptr<Device> dev_;
  KeyBank &bank_;
  RegionCache cache_;
  std::vector<Block> host_;                         // tenant -> page-locked keys
  RegionFences fences_;                             // of the slots
};

// Cached c1 rows of a seeded key bank (B200Server c1_cache): RegionCache::assignByCount decides which tenants hold the bank's c1
// regions, and a fill expands a tenant's c1 rows from the seeds in its bank slot (KeyBank::fillC1) on the store's fill stream,
// ordered against the runs by the regions' RegionFences.  A fill also waits for the fill of the tenant's slot (paging: its images
// must be there).  The rows depend on the seeds only, so a tenant keeps its region while its slot is paged out and back in;
// removing its keys drops it.
class C1Store {
public:
  C1Store(std::shared_ptr<Device> dev, KeyBank &bank, KeyPager *pager)
      : dev_(std::move(dev)), bank_(bank), pager_(pager), cache_(bank.c1Regions()), fences_(dev_, bank.c1Regions()) {}
  // the c1 table entry of every instance of a batch (bank region capacity + h, or -1: draws) whose instances hold bank slots
  // `slots`; the admitted missing tenants' fills are enqueued on the store's stream
  std::vector<int> resolve(const std::vector<int> &tenants, const std::vector<int> &slots) {
    std::vector<RegionCache::Fill> fills;
    std::vector<int> regions = cache_.assignByCount(tenants, fills);
    for (auto &f : fills) {
      const int slot = slots[std::find(tenants.begin(), tenants.end(), f.tenant) - tenants.begin()];
      fences_.awaitReaders(f.region);
      if (pager_) if (void *ev = pager_->fillEvent(slot)) check(evab_stream_wait_event(dev_->ctx(), fences_.stream(), ev));
      bank_.fillC1(f.region, slot, fences_.stream());
      fences_.filled(f.region);
    }
    for (int &r : regions) if (r >= 0) r += bank_.capacity();
    return regions;
  }
  // a run on `stream` with c1 table entries `rows` waits for their regions' fills; once enqueued, it is recorded as their reader
  void beforeRun(void *stream, const int *rows, int n) { fences_.beforeRun(stream, rows, n, bank_.capacity()); }
  void afterRun(void *stream, const int *rows, int n) { fences_.afterRun(stream, rows, n, bank_.capacity()); }
  void drop(int tenant) { cache_.drop(tenant); }
  const RegionCache &cache() const { return cache_; }

private:
  std::shared_ptr<Device> dev_;
  KeyBank &bank_;
  KeyPager *pager_;
  RegionCache cache_;
  RegionFences fences_;   // of the c1 regions
};

// Server-resident input ciphertexts (B200Server store_entries, max_stored, store_storage).  A request names an entry by handle
// where it would carry the ciphertext, and staging copies the entry's device words into the arena (evab_gather_ciphers).  Handles
// increase and are never reused, so a released handle, or one of a tenant whose keys were removed (its entries go with them),
// names nothing afterwards.  Entries do not depend on key residency.
//  - Layout.  "expanded": a device entry holds the size-2 ciphertext [2][ell][N] (2 (k-1) N words).  "seeded" (seeded ciphertexts
//    only): a device entry holds c0 [ell][N] ((k-1) N words) and the Entry keeps the seed; staging adds the seed to the chunk's
//    evab_expand_cipher_uniform call, which draws c1 into the arena exactly as for the same ciphertext sent inline.
//  - Paging (max_stored > store_entries).  Every entry lives in page-locked host memory (a seeded ciphertext as c0 and its seed, in
//    either layout), and the device entries are the regions of a RegionCache keyed by entry id: store() does no device work, and
//    every enqueue resolves its batch's entries (assignAll), filling the missing ones on the fill stream (one upload of the host
//    words; in the expanded layout a seeded entry's c1 is drawn into the region too).  Without paging, entry e is device region e,
//    written by store() and synchronised before it returns.
//  - Ordering, per device region (RegionFences): a fill (or a store() into a released region) waits for the gathers that may still
//    read the region, and a chunk's gather waits for the fills of the regions it reads.
class CipherStore {
public:
  struct Entry {
    int tenant = -1, ell = 0;
    double scale = 0;
    std::uint64_t handle = 0;   // 0: free
    bool seeded = false;        // stored from a seeded ciphertext: `seed` is the seed of its c1
    KeySeed seed{};
    HostBuf host;               // paging: the entry's page-locked words, c0 [ell][N] when seeded, else [2][ell][N]
  };
  // store_storage: "expanded" or "seeded" (true)
  static bool seededLayout(const std::string &storage) {
    if (storage != "expanded" && storage != "seeded")
      throw std::invalid_argument("store_storage must be \"expanded\" or \"seeded\", not \"" + storage + "\"");
    return storage == "seeded";
  }
  // words of a device entry, and of a paged entry's host copy at ell residues
  static std::size_t entryWords(int k, u64 N, bool seededLayout) { return (seededLayout ? 1 : 2) * (std::size_t)(k - 1) * N; }
  static std::size_t hostWords(int ell, u64 N, bool seededCipher) { return (seededCipher ? 1 : 2) * (std::size_t)ell * N; }

  CipherStore(std::shared_ptr<Device> dev, int capacity, int maxStored, bool seeded)
      : dev_(std::move(dev)), seeded_(seeded), entries_(maxStored), cache_(capacity), words_(dev_, (std::size_t)capacity * entryWords()),
        fences_(dev_, capacity) {}
  int capacity() const { return cache_.regions(); }
  int maxStored() const { return (int)entries_.size(); }
  bool paged() const { return maxStored() > capacity(); }
  bool seeded() const { return seeded_; }
  int used() const { return (int)slotOf_.size(); }
  std::size_t entryWords() const { return entryWords(dev_->k(), dev_->N(), seeded_); }
  std::uint64_t fills() const { return paged() ? cache_.fills() : 0; }
  std::uint64_t evictions() const { return paged() ? cache_.evictions() : 0; }
  // the handles whose entry holds a device region (paging: in region order)
  std::vector<std::uint64_t> resident() const {
    std::vector<std::uint64_t> h;
    if (paged()) for (int e : cache_.holders()) h.push_back(entries_[e].handle);
    else for (auto &kv : slotOf_) h.push_back(kv.first);
    return h;
  }
  std::size_t hostBytes() const {
    std::size_t w = 0;
    for (const Entry &e : entries_) w += e.host.size();
    return w * 8;
  }
  // every value of `v` into a free entry of `tenant`, all or nothing.  Without paging, full ciphertexts are uploaded, and seeded
  // ones have their c0 uploaded and (expanded layout) their c1 drawn into the entry once.  With paging the words go to page-locked
  // host memory only.  Returns name -> handle
  std::map<std::string, std::uint64_t> store(int tenant, const B200Valuation &v) {
    const u64 N = dev_->N();
    const int k = dev_->k();
    for (auto &kv : v) {
      const std::string what = "value " + kv.first;
      if (auto *c = std::get_if<HostCipher>(&kv.second)) {
        if (c->size != 2 || c->ell < 1 || c->ell > k - 1 || c->data.size() != (std::size_t)2 * c->ell * N)
          throw std::invalid_argument(what + ": only size-2 ciphertexts of the server's parameters can be stored");
        if (seeded_)
          throw std::invalid_argument(what + " is a full ciphertext: a store with store_storage=\"seeded\" keeps c0 rows and seeds and takes "
                                      "seeded ciphertexts only (B200Secret.encrypt)");
      } else if (auto *sc = std::get_if<HostSeededCipher>(&kv.second)) {
        if (sc->ell < 1 || sc->ell > k - 1 || sc->c0.size() != (std::size_t)sc->ell * N)
          throw std::invalid_argument(what + ": seeded ciphertext does not match the server's parameters (level / degree)");
      } else {
        if (std::holds_alternative<HostCompactCipher>(kv.second)) throw compactRefused(what);
        const char *kind = std::holds_alternative<HostPlain>(kv.second) ? "a plaintext" : std::holds_alternative<StoredCipher>(kv.second) ? "a stored reference" : "a raw vector";
        throw std::invalid_argument(what + " is " + kind + ": only ciphertexts can be stored");
      }
    }
    if (maxStored() - used() < (int)v.size())
      throw std::invalid_argument("the ciphertext store has " + std::to_string(maxStored() - used()) + " free entries of " +
                                  (paged() ? "max_stored=" : "store_entries=") + std::to_string(maxStored()) + " and the valuation holds " +
                                  std::to_string(v.size()) + ": release entries first");
    std::vector<int> ids;
    for (int e = 0; e < maxStored() && ids.size() < v.size(); e++) if (!entries_[e].handle) ids.push_back(e);
    std::vector<HostBuf> host(v.size());
    if (paged()) {   // copied before any entry changes (all or nothing)
      std::size_t i = 0;
      for (auto &kv : v) {
        HostBuf &h = host[i++];
        if (auto *hc = std::get_if<HostCipher>(&kv.second)) h.assign(hc->data.begin(), hc->data.end());
        else { auto &sc = std::get<HostSeededCipher>(kv.second); h.assign(sc.c0.begin(), sc.c0.end()); }
      }
    } else {         // entry e is device region e
      void *stream = fences_.stream();
      std::vector<KeySeed> seeds;
      std::vector<u64 *> c1;
      std::vector<int> ells;
      std::size_t i = 0;
      for (auto &kv : v) {
        const int e = ids[i++];
        u64 *dst = region(e);
        fences_.awaitReaders(e);
        if (auto *hc = std::get_if<HostCipher>(&kv.second)) {
          dev_->upload(dst, hc->data.data(), hc->data.size() * 8, stream);
        } else {
          auto &sc = std::get<HostSeededCipher>(kv.second);
          dev_->upload(dst, sc.c0.data(), sc.c0.size() * 8, stream);
          if (!seeded_) { seeds.push_back(sc.seed); c1.push_back(dst + sc.c0.size()); ells.push_back(sc.ell); }
        }
      }
      if (!seeds.empty()) expandCiphers(*dev_, (int)seeds.size(), seeds.data(), c1.data(), ells.data(), stream);
      check(evab_sync(dev_->ctx(), stream));   // the first request that names an entry needs no fill event
    }
    std::map<std::string, std::uint64_t> out;
    std::size_t i = 0;
    for (auto &kv : v) {
      const int id = ids[i];
      Entry &e = entries_[id];
      e.tenant = tenant; e.handle = next_++; e.host = std::move(host[i++]);
      if (auto *hc = std::get_if<HostCipher>(&kv.second)) { e.ell = hc->ell; e.scale = hc->scale; }
      else { auto &sc = std::get<HostSeededCipher>(kv.second); e.ell = sc.ell; e.scale = sc.scale; e.seeded = true; e.seed = sc.seed; }
      slotOf_[e.handle] = id;
      out[kv.first] = e.handle;
    }
    return out;
  }
  // null: no such entry (never issued, or released)
  const Entry *find(std::uint64_t handle) const {
    auto it = slotOf_.find(handle);
    return it == slotOf_.end() ? nullptr : &entries_[it->second];
  }
  // the device words of a stored ciphertext: its region, as resolved for the batch being enqueued
  const u64 *words(std::uint64_t handle) const {
    const int e = slotOf_.at(handle), r = paged() ? cache_.regionOf(e) : e;
    if (r < 0) throw std::logic_error("stored ciphertext " + std::to_string(handle) + " staged without a device entry (not resolved)");
    return region(r);
  }
  void release(std::uint64_t handle) {
    auto it = slotOf_.find(handle);
    if (it == slotOf_.end()) throw std::invalid_argument("handle " + std::to_string(handle) + " names no stored ciphertext (never issued, or released)");
    clear(it->second);
    slotOf_.erase(it);
  }
  void dropTenant(int tenant) {
    for (auto it = slotOf_.begin(); it != slotOf_.end();)
      if (entries_[it->second].tenant == tenant) { clear(it->second); it = slotOf_.erase(it); }
      else ++it;
  }
  // The device region of every stored reference of the instances inputs[0 .. n), instance b's at [from[b], from[b + 1]) in the
  // order stageInputs meets them (references checked by checkStored).  With paging, the missing entries' fills are enqueued on the
  // fill stream
  std::vector<int> resolve(const B200Valuation *const *inputs, int n, std::vector<int> &from) {
    std::vector<int> ids;
    from.assign(1, 0);
    for (int b = 0; b < n; b++) {
      for (auto &in : *inputs[b])
        if (auto *r = std::get_if<StoredCipher>(&in.second)) ids.push_back(slotOf_.at(r->handle));
      from.push_back((int)ids.size());
    }
    if (!paged() || ids.empty()) return ids;
    std::vector<RegionCache::Fill> fills;
    std::vector<int> regions = cache_.assignAll(ids, fills);
    void *stream = fences_.stream();
    std::vector<KeySeed> seeds;
    std::vector<u64 *> c1;
    std::vector<int> ells;
    for (auto &f : fills) {
      const Entry &e = entries_[f.tenant];
      u64 *dst = region(f.region);
      fences_.awaitReaders(f.region);
      dev_->upload(dst, e.host.data(), e.host.size() * 8, stream);
      if (e.seeded && !seeded_) { seeds.push_back(e.seed); c1.push_back(dst + e.host.size()); ells.push_back(e.ell); }
    }
    if (!seeds.empty()) expandCiphers(*dev_, (int)seeds.size(), seeds.data(), c1.data(), ells.data(), stream);
    for (auto &f : fills) fences_.filled(f.region);
    return regions;
  }
  // a chunk on `stream` that gathers from `regions` waits for their fills; once enqueued, it is recorded as their reader
  void beforeRun(void *stream, const int *regions, int n) { fences_.beforeRun(stream, regions, n); }
  void afterRun(void *stream, const int *regions, int n) { fences_.afterRun(stream, regions, n); }

private:
  u64 *region(int r) const { return words_.get() + (std::size_t)r * entryWords(); }
  // entry e is free again: with paging its device copy is dropped, and its host words freed once no fill reads them
  void clear(int e) {
    if (paged()) {
      cache_.drop(e);
      check(evab_sync(dev_->ctx(), fences_.stream()));
    }
    entries_[e] = Entry();
  }
  std::shared_ptr<Device> dev_;
  bool seeded_;                                     // store_storage="seeded"
  std::vector<Entry> entries_;                      // [max_stored]
  RegionCache cache_;                               // paging: the entry held by each device region
  DBuf words_;                                      // [store_entries][entryWords()]
  RegionFences fences_;                             // of the device regions (destroyed first: its fills read entries_ and write words_)
  std::map<std::uint64_t, int> slotOf_;             // live handle -> entry
  std::uint64_t next_ = 1;
};

// where every instance of a batch reads its keys: its key-bank slot (empty: no key bank) and its c1 table entry (empty: no c1
// cache); and the store regions its stored inputs are gathered from, instance b's stored[storedFrom[b] .. storedFrom[b + 1])
// (storedFrom empty: no store)
struct Residency {
  std::vector<int> slots, c1, stored, storedFrom;
  const int *c1At(int b0) const { return c1.empty() ? nullptr : c1.data() + b0; }
};

struct Shared {
  std::shared_ptr<Device> dev;
  std::unique_ptr<CkksClient> client;
  KeySet keys;
  std::unique_ptr<KeyBank> bank;   // B200Server: the tenants' keys (then `keys` is empty and every batch names a tenant per instance)
  std::unique_ptr<KeyPager> pager; // B200Server with max_tenants > capacity: tenants paged into the bank's regions
  std::unique_ptr<C1Store> c1;     // B200Server with c1_cache > 0: cached c1 rows of a seeded bank (declared after pager: destroyed first)
  std::unique_ptr<CipherStore> store;   // B200Server with store_entries > 0: the tenants' stored input ciphertexts
  std::mutex execMutex;   // serialises execute / executeMany callers of one context (see executeMany), and key-bank changes
  void requireTenant(int t) const { if (pager) pager->requireRegistered(t); else bank->requireOccupied(t); }
  // the residency of every instance, and of the stored inputs of inputs[0 .. n) when given (with paging and a c1 cache: resolved,
  // and the missing fills enqueued: slots, c1 rows, store entries)
  Residency resolve(const std::vector<int> &tenants, const B200Valuation *const *inputs = nullptr, int n = 0) {
    Residency r;
    r.slots = pager ? pager->resolve(tenants) : tenants;
    if (c1) r.c1 = c1->resolve(tenants, r.slots);
    if (store && inputs) r.stored = store->resolve(inputs, n, r.storedFrom);
    return r;
  }
  // the staging and the run on `stream` of instances b0 .. b0 + nb wait for the fills of what they read; once enqueued, they are
  // recorded as its reader
  void beforeRun(void *stream, const Residency &r, int b0, int nb) {
    if (pager) pager->beforeRun(stream, r.slots.data() + b0, nb);
    if (c1) c1->beforeRun(stream, r.c1.data() + b0, nb);
    if (!r.storedFrom.empty()) store->beforeRun(stream, r.stored.data() + r.storedFrom[b0], r.storedFrom[b0 + nb] - r.storedFrom[b0]);
  }
  void afterRun(void *stream, const Residency &r, int b0, int nb) {
    if (pager) pager->afterRun(stream, r.slots.data() + b0, nb);
    if (c1) c1->afterRun(stream, r.c1.data() + b0, nb);
    if (!r.storedFrom.empty()) store->afterRun(stream, r.stored.data() + r.storedFrom[b0], r.storedFrom[b0 + nb] - r.storedFrom[b0]);
  }
};

// SEALPublic::encrypt's checks, slot replication and encoding (reference eva/seal/seal.cpp:24-102), shared by the public-key
// (B200Public) and the secret-key (B200Secret) encryption: Raw inputs are kept, Plain inputs encoded, and every Cipher input's
// device plaintext [ell][N] is handed to `cipher`
inline B200Valuation encodeInputs(Shared &s, const Valuation &inputs, const CKKSSignature &sig,
                                  const std::function<SchemeValue(const u64 *d_pt, int ell, double scale)> &cipher) {
  auto &enc = s.client->encoder();
  const std::size_t slots = enc.slotCount();
  if (slots < (std::size_t)sig.vecSize) throw std::runtime_error("Vector size cannot be larger than slot count");
  if (slots % sig.vecSize) throw std::runtime_error("Vector size must exactly divide the slot count");
  B200Valuation out;
  const u64 N = s.dev->N();
  for (auto &in : inputs) {
    const auto &v = in.second;
    if (v.size() != (std::size_t)sig.vecSize) throw std::runtime_error("Input size does not match program vector size");
    const CKKSEncodingInfo &info = sig.inputs.at(in.first);
    if (info.inputType == Type::Raw) { out[in.first] = std::make_shared<ConstantValue>(sig.vecSize, v); continue; }
    const int ell = s.dev->k() - 1 - info.level;
    if (ell < 1) throw std::runtime_error("input level exceeds the modulus chain");
    std::vector<double> rep;
    rep.reserve(slots);
    for (std::size_t r = slots / v.size(); r > 0; --r) rep.insert(rep.end(), v.begin(), v.end());
    const double scale = std::ldexp(1.0, info.scale);
    DBuf pt(s.dev, (std::size_t)ell * N);
    enc.encode(rep, scale, ell, pt.get());
    if (info.inputType == Type::Cipher) {
      out[in.first] = cipher(pt.get(), ell, scale);
    } else {
      HostPlain h; h.ell = ell; h.scale = scale; h.data.resize((std::size_t)ell * N);
      s.dev->download(h.data.data(), pt.get(), h.data.size() * 8); s.dev->sync();
      out[in.first] = std::move(h);
    }
  }
  return out;
}

// the cached plan of one (program, context) pair; owned by the Program
struct PlanHolder {
  std::shared_ptr<Shared> keepAlive;  // the plan references the context's encoder and keys
  std::unique_ptr<Executor> exec;
  DBuf compactScratch;                // compact_outputs: the replica's compaction work area and packed words, made on first use
  std::uint64_t termCount = 0;
  ExecOptions opt;
};

// a batch that has been enqueued (H2D, plan replays, D2H) and not yet collected: B200Public::submitMany / collect
struct PendingBatch {
  Program *program = nullptr;
  std::vector<const B200Valuation *> inputs;   // the caller keeps them alive until collect()
  std::vector<B200Valuation> outs;
  std::vector<void *> streams;
  std::vector<std::shared_ptr<PlanHolder>> plans;   // the plans it runs on stay alive until it is collected (set_options may replace them meanwhile)
  std::vector<int> tenants;                         // key-bank tenant of every instance (B200Server), empty with a single key set
  int compact = 0;                                  // compact_outputs precision at submit (0: full outputs); collect's redo keeps it
  int slot = 0;
  bool collected = false;
  std::shared_ptr<Shared> keep;
  // dropped without collect(): the copies into `outs` must not outlive their buffers
  ~PendingBatch() { if (!collected && keep) for (void *st : streams) keep->dev->sync(st); }
};

class B200Public {
public:
  explicit B200Public(std::shared_ptr<Shared> s) : s_(std::move(s)) {
    static std::atomic<std::uint64_t> next{1};
    id_ = next.fetch_add(1);
  }

  // SEALPublic::encrypt -- reference eva/seal/seal.cpp:24-102
  B200Valuation encrypt(const Valuation &inputs, const CKKSSignature &sig) {
    return encodeInputs(*s_, inputs, sig, [&](const u64 *pt, int ell, double scale) -> SchemeValue {
      DBuf ct = s_->client->encrypt(s_->keys, pt, ell);
      HostCipher h; h.size = 2; h.ell = ell; h.scale = scale; h.data.resize((std::size_t)2 * ell * s_->dev->N());
      s_->dev->download(h.data.data(), ct.get(), h.data.size() * 8); s_->dev->sync();
      return h;
    });
  }

  // one plan (arena, streams, captured graph) per (context, batch, replica); replicas of the same
  // batch size run concurrently in executeMany
  std::uint64_t planKey(int batch, int replica) const { return (id_ << 32) | ((std::uint64_t)replica << 16) | (std::uint64_t)batch; }
  Executor &executorFor(Program &program, int batch = 1, int replica = 0) { return *holderFor(program, batch, replica)->exec; }
  std::shared_ptr<PlanHolder> holderFor(Program &program, int batch = 1, int replica = 0) {
    if (batch < 1 || batch > 65535 || replica < 0 || replica > 65535) throw std::invalid_argument("batch / replica out of range");
    const std::uint64_t key = planKey(batch, replica);
    auto h = std::static_pointer_cast<PlanHolder>(program.attachment(key));
    if (!h || h->termCount != program.termCount() || h->opt.hoistModUp != options.hoistModUp || h->opt.approxHoist != options.approxHoist || h->opt.rotationChunk != options.rotationChunk ||
        h->opt.rotationSums != options.rotationSums ||
        h->opt.arenaLimit != options.arenaLimit) {   // stale plan: rebuilt
      h = std::make_shared<PlanHolder>();
      h->keepAlive = s_;
      ExecOptions o = options;
      o.batch = batch;
      h->opt = o;   // as requested (what the staleness test above compares)
      h->exec = std::make_unique<Executor>(s_->dev, s_->keys, program, o, s_->bank.get());
      h->termCount = program.termCount();
      plansBuilt++;
      program.attach(key, h);
    }
    return h;
  }
  void dropExecutor(Program &program, int batch = 1, int replica = 0) { program.attach(planKey(batch, replica), nullptr); }

  // upload the host inputs of a chunk's nb valuations into the executor's arena (instance b from inputs[b]; H2D on `stream`).
  // Client-supplied valuations are untrusted (they may come from a file): every buffer is checked against the shape the plan
  // expects before its copy.  A seeded ciphertext's c0 is uploaded like any other input; the c1 rows of all of the chunk's seeded
  // ciphertexts are then expanded on the device by one evab_expand_cipher_uniform call.  The chunk's stored inputs (references
  // checked by checkStored and resolved before the batch was enqueued) are copied from the store by one evab_gather_ciphers call:
  // whole entries, or with store_storage="seeded" their c0 rows, whose seeds join the expansion call.
  void stageInputs(Executor &ex, Program &program, const B200Valuation *const *inputs, int nb, void *stream) {
    const u64 N = s_->dev->N();
    std::vector<KeySeed> seeds;
    std::vector<u64 *> c1;
    std::vector<int> ells;
    std::vector<const u64 *> gatherSrc;
    std::vector<u64 *> gatherDst;
    std::vector<u64> gatherWords;
    for (int b = 0; b < nb; b++)
      for (auto &in : *inputs[b]) {
        auto term = program.getInput(in.first);
        const ValueInfo &vi = ex.info(term);
        if (auto *c = std::get_if<HostCipher>(&in.second)) {
          if (vi.kind != Kind::Cipher || c->ell != vi.ell || c->size != vi.size || c->data.size() != (std::size_t)vi.size * vi.ell * N)
            throw std::runtime_error("input " + in.first + ": ciphertext does not match the program signature");
          s_->dev->upload(ex.valuePtr(term, b), c->data.data(), c->data.size() * 8, stream);
        } else if (auto *sc = std::get_if<HostSeededCipher>(&in.second)) {
          if (vi.kind != Kind::Cipher || vi.size != 2 || sc->ell != vi.ell || sc->c0.size() != (std::size_t)vi.ell * N)
            throw std::runtime_error("input " + in.first + ": seeded ciphertext does not match the program signature");
          u64 *dst = ex.valuePtr(term, b);
          s_->dev->upload(dst, sc->c0.data(), sc->c0.size() * 8, stream);
          seeds.push_back(sc->seed); c1.push_back(dst + sc->c0.size()); ells.push_back(sc->ell);
        } else if (auto *r = std::get_if<StoredCipher>(&in.second)) {
          const CipherStore::Entry *e = s_->store ? s_->store->find(r->handle) : nullptr;
          if (!e) throw std::logic_error("input " + in.first + ": stored reference staged without checkStored");
          u64 *dst = ex.valuePtr(term, b);
          const std::size_t c0 = (std::size_t)vi.ell * N;
          gatherSrc.push_back(s_->store->words(r->handle)); gatherDst.push_back(dst);
          if (s_->store->seeded()) {
            gatherWords.push_back(c0);
            seeds.push_back(e->seed); c1.push_back(dst + c0); ells.push_back(vi.ell);
          } else {
            gatherWords.push_back(2 * c0);
          }
        } else if (std::holds_alternative<HostCompactCipher>(in.second)) {
          throw compactRefused("input " + in.first);
        } else if (auto *p = std::get_if<HostPlain>(&in.second)) {
          if (vi.kind != Kind::Plain || p->ell != vi.ell || p->data.size() != (std::size_t)vi.ell * N)
            throw std::runtime_error("input " + in.first + ": plaintext does not match the program signature");
          s_->dev->upload(ex.valuePtr(term, b), p->data.data(), (std::size_t)p->ell * N * 8, stream);
        } else {
          if (vi.kind != Kind::Raw) throw std::runtime_error("input " + in.first + ": raw vector does not match the program signature");
          auto &cv = std::get<std::shared_ptr<ConstantValue>>(in.second);
          std::vector<double> x;
          cv->expandTo(x, program.getVecSize());
          ex.setRawInput(in.first, x, b);
        }
      }
    // One launch for the chunk, on the chunk's stream, before its run.  Stream order gives the rest: the expansion starts after the
    // replica's previous run has stopped reading the arena, a collect() redo (the zero-digit case) stages again and so expands the
    // same words again, and a packed arena never lends an input's storage to another value (inputs are pinned).  The same holds
    // for the gather of stored inputs, whose entries cannot be released while a batch that names them is uncollected; the caller
    // orders it against the fills of the entries' device regions (Shared::beforeRun / afterRun).
    if (!seeds.empty()) expandCiphers(*s_->dev, (int)seeds.size(), seeds.data(), c1.data(), ells.data(), stream);
    if (!gatherSrc.empty())
      check(evab_gather_ciphers(s_->dev->ctx(), (int)gatherSrc.size(), gatherSrc.data(), gatherDst.data(), gatherWords.data(), stream));
  }
  // Stored inputs come from outside the program as much as inline ones.  Before anything of a batch is enqueued, every reference
  // is checked: the handle names an entry, the entry belongs to the tenant of the instance that names it (tenants[b]; null without
  // a key bank), and its level and size are the input's in the plan, as stageInputs checks an inline ciphertext.  With paging, the
  // batch names at most store_entries distinct entries (all of them are on the device while it is staged)
  void checkStored(const Executor &ex, Program &program, const B200Valuation *const *inputs, const int *tenants, int nb) const {
    std::set<std::uint64_t> distinct;
    for (int b = 0; b < nb; b++)
      for (auto &in : *inputs[b]) {
        auto *r = std::get_if<StoredCipher>(&in.second);
        if (!r) continue;
        const std::string what = "input " + in.first + " (stored ciphertext, handle " + std::to_string(r->handle) + ")";
        if (!s_->store || !tenants) throw std::invalid_argument(what + ": this context has no ciphertext store (a B200Server with store_entries > 0 has one)");
        const std::string who = " of tenant " + std::to_string(tenants[b]);
        const CipherStore::Entry *e = s_->store->find(r->handle);
        if (!e) throw std::invalid_argument(what + who + ": no such entry (never issued, released, or its tenant's keys were removed)");
        if (e->tenant != tenants[b]) throw std::invalid_argument(what + who + ": the entry belongs to another tenant");
        const ValueInfo &vi = ex.info(program.getInput(in.first));
        if (vi.kind != Kind::Cipher || vi.size != 2 || vi.ell != e->ell)
          throw std::invalid_argument(what + who + ": the stored ciphertext (size 2, ell " + std::to_string(e->ell) + ") does not match the program signature (" +
                                      (vi.kind == Kind::Cipher ? "size " + std::to_string(vi.size) + ", ell " + std::to_string(vi.ell) : std::string("not a ciphertext")) + ")");
        distinct.insert(r->handle);
      }
    if (s_->store && (int)distinct.size() > s_->store->capacity())
      throw std::invalid_argument("a batch names " + std::to_string(distinct.size()) + " distinct stored ciphertexts but the store has store_entries=" +
                                  std::to_string(s_->store->capacity()) + " device entries (max_stored=" + std::to_string(s_->store->maxStored()) +
                                  "): split the batch");
  }
  // with execMutex held: does a submitted, not yet collected batch name this stored ciphertext?
  bool storedInFlightLocked(std::uint64_t handle) const {
    for (auto &w : inFlight_)
      if (auto p = w.lock(); p && !p->collected)
        for (const B200Valuation *v : p->inputs)
          for (auto &in : *v)
            if (auto *r = std::get_if<StoredCipher>(&in.second); r && r->handle == handle) return true;
    return false;
  }
  // plans and arenas are cached on the Program: a call that omits an input would silently compute on the previous
  // call's ciphertext.  The reference builds a fresh executor per call and fails on the missing value
  // (seal_executor.h:264); so does this.
  static void requireAllInputs(Program &program, const B200Valuation &inputs) {
    for (auto &in : program.getInputs()) {
      auto it = inputs.values.find(in.first);
      if (it == inputs.values.end()) throw std::runtime_error("Missing input value: " + in.first);
      if (std::holds_alternative<HostCompactCipher>(it->second)) throw compactRefused("input " + in.first);
    }
  }
  // SEALPublic::execute -- reference eva/seal/seal.cpp:104-122.  Host buffers in,
  // host buffers out: H2D of the inputs, the DAG on the GPU, D2H of the outputs.
  B200Valuation execute(Program &program, const B200Valuation &inputs) {
    std::vector<const B200Valuation *> in{&inputs};
    return std::move(executeMany(program, in)[0]);
  }
  // Batched execute: N valuations of the same program run as ONE plan replay whose kernels
  // each cover all instances (horizontal fusion; SURVEY.md 8f-3).  Results are identical
  // to N separate execute() calls.
  std::vector<B200Valuation> executeBatch(Program &program, const std::vector<B200Valuation> &inputs) {
    std::vector<const B200Valuation *> in;
    for (auto &v : inputs) in.push_back(&v);
    return executeMany(program, in);
  }
  // B valuations are split into chunks of options.fuse instances; every chunk has its own plan
  // replica (arena + captured graph) and all replicas are in flight at once: H2D, graph and D2H of
  // different chunks overlap, and the SMs are filled by concurrency rather than by launch width.
  std::vector<B200Valuation> executeMany(Program &program, const std::vector<const B200Valuation *> &inputs, int compact = -1) {
    auto p = submitMany(program, inputs, 0, {}, compact);
    return collect(*p);
  }
  // Pipelined form of executeMany: submitMany enqueues a batch (H2D of its inputs, the plan replays, D2H of its outputs) and returns;
  // collect waits for it and hands out the results.  Batches submitted with different `slot` numbers (0..7) use disjoint plan
  // replicas, so the head of one overlaps the tail of the other (each batch alone ramps up replica by replica and drains the same way).
  // tenants: with a key bank (B200Server), the tenant whose keys instance b runs with; otherwise empty
  // compact: the compact_outputs precision of this batch (-1: the context's option)
  std::shared_ptr<PendingBatch> submitMany(Program &program, const std::vector<const B200Valuation *> &inputs, int slot = 0, std::vector<int> tenants = {},
                                           int compact = -1) {
    if (inputs.empty()) throw std::invalid_argument("execute needs at least one valuation");
    if (slot < 0 || slot > 7) throw std::invalid_argument("slot out of range (0..7)");
    if (s_->bank ? tenants.size() != inputs.size() : !tenants.empty()) throw std::invalid_argument("one tenant per valuation on a key bank, none otherwise");
    for (auto *v : inputs) requireAllInputs(program, *v);
    // one caller at a time per context: plan replicas own single arenas and raw-input buffers (the reference's
    // execute is re-entrant because it builds a new executor per call; concurrent callers are serialised here)
    std::lock_guard<std::mutex> guard(s_->execMutex);
    for (int t : tenants) s_->requireTenant(t);
    if (auto prev = inFlight_[slot].lock(); prev && !prev->collected) throw std::runtime_error("slot in use: collect the batch submitted before");
    auto p = std::make_shared<PendingBatch>();
    p->program = &program; p->inputs = inputs; p->slot = slot; p->keep = s_; p->tenants = std::move(tenants);
    p->compact = compact < 0 ? compactOutputs : compact;
    enqueueLocked(*p);
    inFlight_[slot] = p;
    return p;
  }
  std::vector<B200Valuation> collect(PendingBatch &p) {
    if (p.collected) throw std::runtime_error("this batch has been collected already");
    std::lock_guard<std::mutex> guard(s_->execMutex);
    p.collected = true;
    for (void *st : p.streams) s_->dev->sync(st);
    bool redo = false;
    for (auto &h : p.plans) if (h->exec->flagsRaised()) redo = true;
    if (redo) {
      // a digit of a rotated ciphertext held a zero coefficient: the shared mod-up of that rotation group is not SEAL's value
      // (ops_impl.hpp hoisted_modup).  Redo the call on plans without it -- exact, and from now on for this context.
      if (verbosity() >= 1) std::fprintf(stderr, "EVA: zero digit coefficient met; rotation groups of this context no longer share their mod-up\n");
      options.hoistModUp = false;      // executorFor rebuilds every plan whose option differs
      p.outs.clear(); p.streams.clear(); p.plans.clear();
      enqueueLocked(p);
      for (void *st : p.streams) s_->dev->sync(st);
    }
    return std::move(p.outs);
  }
  static constexpr int kSlotReplicas = 4096;   // replica numbers of slot s: s * kSlotReplicas + r
  void enqueueLocked(PendingBatch &p) {
    Program &program = *p.program;
    const std::vector<const B200Valuation *> &inputs = p.inputs;
    const int B = (int)inputs.size();
    const int F = std::max(1, std::min(options.fuse, B));
    const int base = p.slot * kSlotReplicas;
    std::vector<B200Valuation> &outs = p.outs;
    outs.assign(B, B200Valuation());
    std::vector<void *> &streams = p.streams;
    const u64 N = s_->dev->N();
    static const bool trace = std::getenv("EVAB_TRACE") != nullptr;
    auto now = [] { return std::chrono::steady_clock::now(); };
    double tPlan = 0, tStage = 0, tRun = 0;
    auto t00 = now();
    // replicas are bounded by device memory (an arena each): with R replicas chunk g runs on replica g % R
    // after that replica's previous chunk has completed (its outputs are already on their way to the host)
    int R = std::min((B + F - 1) / F, kSlotReplicas);
    {
      Executor &first = executorFor(program, std::min(F, B), base);
      std::size_t have = 1;   // the slot's first replica exists; count the ones already built for this program
      while ((int)have < R && program.attachment(planKey(std::min(F, B), base + (int)have))) have++;
      if ((int)have < R) {    // new arenas are needed: how many fit?  (cudaMemGetInfo is slow: never on the steady path)
        std::size_t freeB = 0, totalB = 0;
        check(evab_mem_info(s_->dev->ctx(), &freeB, &totalB));
        const std::size_t per = std::max<std::size_t>(first.arenaBytes(), 1);
        const std::size_t extra = (std::size_t)(0.8 * (double)freeB) / per;
        R = (int)std::max<std::size_t>(1, std::min<std::size_t>((std::size_t)R, have + extra));
      }
      if (const char *cap = std::getenv("EVAB_MAX_REPLICAS")) R = std::max(1, std::min(R, std::atoi(cap)));   // tests / tuning
      checkStored(first, program, inputs.data(), p.tenants.empty() ? nullptr : p.tenants.data(), B);
    }
    std::vector<char> busy(R, 0);
    // residency of every instance and stored input, resolved at every enqueue (so that collect's redo refills a tenant or a stored
    // ciphertext evicted meanwhile)
    const Residency res = s_->resolve(p.tenants, inputs.data(), B);
    for (int b0 = 0, g = 0; b0 < B; b0 += F, g++) {
      const int nb = std::min(F, B - b0);
      const int r = g % R;
      auto t0 = now();
      std::shared_ptr<PlanHolder> holder = holderFor(program, nb, base + r);
      Executor &ex = *holder->exec;
      void *st = ex.mainStream();
      if (busy[r]) s_->dev->sync(st);   // the replica's arena is reused: wait for its previous chunk
      busy[r] = 1;
      if (!res.slots.empty()) ex.setKeyTable(res.slots.data() + b0, res.c1At(b0), nb);
      if (std::find(streams.begin(), streams.end(), st) == streams.end()) streams.push_back(st);
      if (std::find(p.plans.begin(), p.plans.end(), holder) == p.plans.end()) p.plans.push_back(holder);
      auto t1 = now();
      s_->beforeRun(st, res, b0, nb);
      stageInputs(ex, program, inputs.data() + b0, nb, st);
      auto t2 = now();
      ex.run(st);
      s_->afterRun(st, res, b0, nb);
      if (p.compact) compactOutputsOf(*holder, program, p.compact, outs.data() + b0, nb, st);
      auto t3 = now();
      tPlan += std::chrono::duration<double>(t1 - t0).count(); tStage += std::chrono::duration<double>(t2 - t1).count();
      tRun += std::chrono::duration<double>(t3 - t2).count();
      for (int b = 0; b < nb; b++)
        for (auto &o : program.getOutputs()) {
          const ValueInfo &vi = ex.info(o.second);
          B200Valuation &out = outs[b0 + b];
          if (out.values.count(o.first)) continue;   // compacted
          if (vi.kind == Kind::Cipher) {
            HostCipher h; h.size = vi.size; h.ell = vi.ell; h.scale = vi.scale; h.data.resize((std::size_t)vi.size * vi.ell * N);
            s_->dev->download(h.data.data(), ex.valuePtr(o.second, b), h.data.size() * 8, st);
            out[o.first] = std::move(h);
          } else if (vi.kind == Kind::Plain) {
            HostPlain h; h.ell = vi.ell; h.scale = vi.scale; h.data.resize((std::size_t)vi.ell * N);
            s_->dev->download(h.data.data(), ex.valuePtr(o.second, b), h.data.size() * 8, st);
            out[o.first] = std::move(h);
          } else {
            out[o.first] = std::make_shared<ConstantValue>(program.getVecSize(), ex.rawValue(o.second->index, b));
          }
        }
    }
    if (trace)
      std::fprintf(stderr, "[evab] enqueue B=%d F=%d slot=%d: plan %.3f stage %.3f run %.3f enqueue-total %.3f ms\n", B, F, p.slot, tPlan * 1e3, tStage * 1e3, tRun * 1e3,
                   std::chrono::duration<double>(now() - t00).count() * 1e3);
  }
  // compact responses of a chunk of nb instances just run on `st` by the replica `h`: every output that compactShape compacts at
  // precision p is switched and packed on the device by one evab_compact_ciphers call over the chunk, then only its packed words are
  // downloaded into outs[b][name].  The scratch is the replica's own (no allocation on the steady path; nothing while the option is
  // off): its chunks run in order on `st`, and each output's downloads are enqueued before the next compaction rewrites the words
  void compactOutputsOf(PlanHolder &h, Program &program, int p, B200Valuation *outs, int nb, void *st) {
    const u64 N = s_->dev->N();
    evab_ctx *ctx = s_->dev->ctx();
    Executor &ex = *h.exec;
    for (auto &o : program.getOutputs()) {
      const ValueInfo &vi = ex.info(o.second);
      const CompactShape cs = compactShape(s_->dev->primes(), vi.kind == Kind::Cipher, vi.size, vi.ell, vi.scale, o.second->range, p, N);
      if (!cs.compact) continue;
      const std::size_t W = (N * cs.bits + 63) / 64;
      const std::size_t workWords = evab_compact_work_bytes(ctx, nb, vi.ell) / 8, need = workWords + (std::size_t)nb * 2 * W;
      if (h.compactScratch.words() < need) {
        s_->dev->sync(st);                        // the replica's earlier chunks may still use the old area
        h.compactScratch = DBuf();
        h.compactScratch = DBuf(s_->dev, need);
        s_->dev->sync();                          // allocated before `st` uses it
      }
      u64 *work = h.compactScratch.get(), *dst = work + workWords;
      std::vector<const u64 *> src(nb);
      std::vector<u64 *> to(nb);
      for (int b = 0; b < nb; b++) { src[b] = ex.valuePtr(o.second, b); to[b] = dst + (std::size_t)b * 2 * W; }
      check(evab_compact_ciphers(ctx, nb, src.data(), to.data(), vi.ell, cs.shift, cs.bits, work, st));
      for (int b = 0; b < nb; b++) {
        HostCompactCipher hc; hc.bits = cs.bits; hc.scale = cs.scale; hc.words.resize(2 * W);
        s_->dev->download(hc.words.data(), to[b], 2 * W * 8, st);
        outs[b][o.first] = std::move(hc);
      }
    }
  }
  // with execMutex held: does a submitted, not yet collected batch run an instance with this tenant's keys?
  bool tenantInFlightLocked(int t) const {
    for (auto &w : inFlight_)
      if (auto p = w.lock(); p && !p->collected && std::find(p->tenants.begin(), p->tenants.end(), t) != p->tenants.end()) return true;
    return false;
  }
  std::shared_ptr<Shared> shared() const { return s_; }
  ExecOptions options;
  int compactOutputs = 0;         // compact responses: bits of precision after the binary point (0: off); shapes no plan
  std::uint64_t plansBuilt = 0;   // executors constructed by this context (plan build + arena + graph capture each)

private:
  std::shared_ptr<Shared> s_;
  std::uint64_t id_ = 0;
  std::weak_ptr<PendingBatch> inFlight_[8];
};

// One device and one parameter set serving many clients: each client's evaluation keys are a tenant of a key bank, the plans of
// a program belong to the server (built, allocated and captured once, whatever the number of tenants), and every instance of a
// batch runs with its own tenant's keys.  Execution is B200Public's (replicas, slots, fused chunks, the zero-digit redo).
class B200Server {
public:
  // maxTenants < 0 or == capacity: tenant id = bank region, filled when the keys are added.  maxTenants > capacity: paging (KeyPager)
  // rotationKeys: the bank's Galois keys (rotationKeySteps); rotations without a key of their own are composed.
  // hoistConstants: "stored" -- every region holds the hoist constants of its keys; "inline" -- keys only, the constants are formed
  // inside the key-switch inner products (KeyBank).  keyStorage: "expanded" -- every key in full; "seeded" (inline constants only) --
  // c0 rows and seeds, the key switches draw the c1 rows (KeyBank).  c1Cache (seeded keys, 0 .. capacity): regions holding the
  // expanded c1 rows of the tenants used most (C1Store); 0 is the plain seeded bank
  // storeEntries: device entries of the ciphertext store (CipherStore), 0 for none.  maxStored < 0 or == storeEntries: every stored
  // ciphertext holds a device entry; maxStored > storeEntries: up to maxStored in page-locked host memory, paged into the device
  // entries.  storeStorage: "expanded" -- device entries hold whole ciphertexts; "seeded" -- c0 rows and seeds of seeded ciphertexts
  B200Server(const CKKSParameters &params, int capacity, int device, int maxTenants = -1, const std::string &rotationKeys = "program",
             const std::string &hoistConstants = "stored", const std::string &keyStorage = "expanded", int c1Cache = 0, int storeEntries = 0,
             int maxStored = -1, const std::string &storeStorage = "expanded")
      : rotationKeys_(rotationKeys), hoistConstants_(hoistConstants), keyStorage_(keyStorage), storeStorage_(storeStorage) {
    if (storeEntries < 0) throw std::invalid_argument("store_entries (" + std::to_string(storeEntries) + ") must be >= 0");
    const bool seededStore = CipherStore::seededLayout(storeStorage);
    if (maxStored >= 0 && maxStored < storeEntries)
      throw std::invalid_argument("max_stored (" + std::to_string(maxStored) + ") is below the number of device entries (store_entries " +
                                  std::to_string(storeEntries) + ")");
    if (maxStored > 0 && storeEntries == 0)
      throw std::invalid_argument("max_stored (" + std::to_string(maxStored) + ") pages stored ciphertexts into device entries: it needs store_entries > 0");
    if (hoistConstants != "stored" && hoistConstants != "inline")
      throw std::invalid_argument("hoist_constants must be \"stored\" or \"inline\", not \"" + hoistConstants + "\"");
    if (keyStorage != "expanded" && !(keyStorage == "seeded" && hoistConstants == "inline"))
      throw std::invalid_argument("key_storage must be \"expanded\", or \"seeded\" with hoist_constants=\"inline\" (got key_storage=\"" +
                                  keyStorage + "\", hoist_constants=\"" + hoistConstants + "\")");
    if (c1Cache < 0 || c1Cache > capacity)
      throw std::invalid_argument("c1_cache (" + std::to_string(c1Cache) + ") must be in [0, capacity] (capacity " + std::to_string(capacity) + ")");
    if (c1Cache > 0 && keyStorage != "seeded")
      throw std::invalid_argument("c1_cache (" + std::to_string(c1Cache) + ") caches the c1 rows of seeded keys: it needs key_storage=\"seeded\" (got key_storage=\"" +
                                  keyStorage + "\")");
    if (maxTenants >= 0 && maxTenants < capacity)
      throw std::invalid_argument("max_tenants (" + std::to_string(maxTenants) + ") is below the number of device slots (capacity " + std::to_string(capacity) + ")");
    const std::vector<int> steps = rotationKeySteps(params, rotationKeys);
    std::vector<int> bits(params.primeBits.begin(), params.primeBits.end());
    auto s = std::make_shared<Shared>();
    s->dev = std::make_shared<Device>(params.polyModulusDegree, hmod::createCoeffModulus(params.polyModulusDegree, bits), device);
    s->client = std::make_unique<CkksClient>(s->dev, 0);
    std::set<u64> elts;
    for (int step : steps) {
      const u64 elt = evab_galois_elt_from_step(params.polyModulusDegree, step);
      if (!elt) throw std::invalid_argument("step count too large");
      elts.insert(elt);
    }
    s->bank = std::make_unique<KeyBank>(s->dev, elts, capacity, hoistConstants == "inline", keyStorage == "seeded", c1Cache);
    if (maxTenants > capacity) s->pager = std::make_unique<KeyPager>(s->dev, *s->bank, maxTenants);
    if (c1Cache > 0) s->c1 = std::make_unique<C1Store>(s->dev, *s->bank, s->pager.get());
    if (storeEntries > 0) s->store = std::make_unique<CipherStore>(s->dev, storeEntries, std::max(maxStored, storeEntries), seededStore);
    pub_ = std::make_unique<B200Public>(s);
  }
  // the ciphertexts of `enc` (full or seeded; seeded only with store_storage="seeded") into the store as `tenant`'s entries, all or
  // nothing: name -> handle.  With paging into host memory only (no device work)
  std::map<std::string, std::uint64_t> store(int tenant, const B200Valuation &enc) {
    std::lock_guard<std::mutex> guard(shared()->execMutex);
    requireStore();
    shared()->requireTenant(tenant);
    return shared()->store->store(tenant, enc);
  }
  void release(std::uint64_t handle) {
    std::lock_guard<std::mutex> guard(shared()->execMutex);
    requireStore();
    if (pub_->storedInFlightLocked(handle))   // collect's redo stages the batch's inputs again
      throw std::runtime_error("stored ciphertext " + std::to_string(handle) + " is used by a batch that has not been collected");
    shared()->store->release(handle);
  }
  const CipherStore *cipherStore() const { return shared()->store.get(); }
  // host images [k-1][2][k][N] (shapes checked by the caller); every element of the rotation set must be present
  int addKeys(const u64 *relin, const std::map<u64, const u64 *> &galois) {
    if (bank().seededKeys())
      throw std::invalid_argument("this server was built with key_storage=\"seeded\" and takes compressed keys only: add_compressed_keys, or "
                                  "add_keys of a context whose keys have seeds (generate_keys)");
    for (u64 e : bank().elements())
      if (!galois.count(e)) throw std::invalid_argument("Galois key for element " + std::to_string(e) + " of the server's rotation set is missing");
    std::lock_guard<std::mutex> guard(shared()->execMutex);
    return shared()->pager ? shared()->pager->add(relin, galois) : shared()->bank->add(relin, galois);
  }
  // compressed keys: host c0 rows [k-1][k][N] and 32-byte seeds (shapes checked by the caller); the c1 rows are expanded on the device
  int addCompressedKeys(const u64 *relinC0, const KeySeed &relinSeed, const std::map<u64, std::pair<const u64 *, KeySeed>> &galois) {
    for (u64 e : bank().elements())
      if (!galois.count(e)) throw std::invalid_argument("Galois key for element " + std::to_string(e) + " of the server's rotation set is missing");
    std::lock_guard<std::mutex> guard(shared()->execMutex);
    if (shared()->pager) return shared()->pager->addCompressed(relinC0, relinSeed, galois);
    std::vector<u64> image(bank().compressedWords());
    bank().packCompressed(image.data(), relinC0, relinSeed, galois);
    return shared()->bank->addCompressed(image.data());
  }
  void removeKeys(int t) {
    std::lock_guard<std::mutex> guard(shared()->execMutex);
    shared()->requireTenant(t);
    if (pub_->tenantInFlightLocked(t)) throw std::runtime_error("tenant " + std::to_string(t) + " is used by a batch that has not been collected");
    if (shared()->c1) shared()->c1->drop(t);   // an id reused with new keys never reads this tenant's rows
    if (shared()->store) shared()->store->dropTenant(t);   // nor its stored ciphertexts
    if (shared()->pager) shared()->pager->remove(t);
    else shared()->bank->remove(t);
  }
  // device-resident hooks: stage a plan replica's inputs for (tenant, valuation) requests, and run it.  With paging, run resolves the
  // staged tenants again (a tenant evicted since is filled again) and waits / records as enqueueLocked does
  void stageInputs(Program &prog, const std::vector<std::pair<int, const B200Valuation *>> &rq, void *stream, int replica) {
    std::vector<int> tenants;
    for (auto &r : rq) tenants.push_back(r.first);
    std::lock_guard<std::mutex> guard(shared()->execMutex);
    for (int t : tenants) shared()->requireTenant(t);
    Executor &ex = pub_->executorFor(prog, (int)rq.size(), replica);
    std::vector<const B200Valuation *> in;
    for (auto &r : rq) in.push_back(r.second);
    pub_->checkStored(ex, prog, in.data(), tenants.data(), (int)in.size());
    staged_[&ex] = tenants;
    const Residency res = shared()->resolve(tenants, in.data(), (int)in.size());
    setKeyTable(ex, res, stream);
    shared()->beforeRun(stream, res, 0, (int)in.size());
    pub_->stageInputs(ex, prog, in.data(), (int)in.size(), stream);
    shared()->afterRun(stream, res, 0, (int)in.size());
  }
  // tenants: replaces the staged tenants of the replica (same count)
  void runResident(Program &prog, void *stream, int batch, int replica, const std::vector<int> &tenants = {}) {
    std::lock_guard<std::mutex> guard(shared()->execMutex);
    Executor &ex = pub_->executorFor(prog, batch, replica);
    if (!tenants.empty()) {
      if ((int)tenants.size() != batch) throw std::invalid_argument("run_resident: one tenant per instance");
      for (int t : tenants) shared()->requireTenant(t);
      staged_[&ex] = tenants;
    }
    KeyPager *pager = shared()->pager.get();
    auto it = staged_.find(&ex);
    if (!pager && it == staged_.end()) { ex.run(stream); return; }
    if (it == staged_.end()) throw std::runtime_error("run_resident: stage the replica's inputs first");
    if (pager) for (int t : it->second) pager->requireRegistered(t);
    const Residency res = shared()->resolve(it->second);
    setKeyTable(ex, res, stream);
    shared()->beforeRun(stream, res, 0, batch);
    ex.run(stream);
    shared()->afterRun(stream, res, 0, batch);
  }
  std::shared_ptr<PendingBatch> submit(Program &program, const std::vector<std::pair<int, const B200Valuation *>> &requests, int slot = 0) {
    std::vector<const B200Valuation *> in;
    std::vector<int> tenants;
    for (auto &r : requests) { tenants.push_back(r.first); in.push_back(r.second); }
    return pub_->submitMany(program, in, slot, std::move(tenants));
  }
  std::vector<B200Valuation> executeBatch(Program &program, const std::vector<std::pair<int, const B200Valuation *>> &requests) {
    auto p = submit(program, requests, 0);
    return pub_->collect(*p);
  }
  B200Public &pub() { return *pub_; }
  const KeyBank &bank() const { return *pub_->shared()->bank; }
  const std::string &rotationKeys() const { return rotationKeys_; }
  const std::string &hoistConstants() const { return hoistConstants_; }
  const std::string &keyStorage() const { return keyStorage_; }
  const std::string &storeStorage() const { return storeStorage_; }
  std::shared_ptr<Shared> shared() const { return pub_->shared(); }

private:
  void requireStore() const {
    if (!shared()->store) throw std::invalid_argument("this server has no ciphertext store: build it with store_entries > 0");
  }
  // the executor's page-locked key table is read by its previous run's stream-ordered upload: rewritten only after that run
  void setKeyTable(Executor &ex, const Residency &res, void *stream) {
    const int n = (int)res.slots.size();
    if (ex.keyTableIs(res.slots.data(), res.c1At(0), n)) return;
    shared()->dev->sync(stream);
    ex.setKeyTable(res.slots.data(), res.c1At(0), n);
  }
  std::string rotationKeys_, hoistConstants_, keyStorage_, storeStorage_;
  std::unique_ptr<B200Public> pub_;
  std::map<const Executor *, std::vector<int>> staged_;   // device-resident hooks: the tenants staged on a plan replica
};

class B200Secret {
public:
  explicit B200Secret(std::shared_ptr<Shared> s) : s_(std::move(s)) {}
  // Encryptor::encrypt_symmetric (SEAL's seed-compressed Serializable<Ciphertext>): B200Public::encrypt's checks and encoding, every
  // Cipher input a seeded ciphertext (c0 and the seed of c1, half the bytes).  Only the holder of the secret key can make one
  B200Valuation encrypt(const Valuation &inputs, const CKKSSignature &sig) {
    if (!s_->keys.sk) throw std::runtime_error("this context has no secret key");
    return encodeInputs(*s_, inputs, sig, [&](const u64 *pt, int ell, double scale) -> SchemeValue {
      auto ct = s_->client->encryptSeeded(s_->keys, pt, ell);
      HostSeededCipher h; h.ell = ell; h.scale = scale; h.seed = ct.second; h.c0.resize((std::size_t)ell * s_->dev->N());
      s_->dev->download(h.c0.data(), ct.first.get(), h.c0.size() * 8); s_->dev->sync();
      return h;
    });
  }
  // SEALSecret::decrypt -- reference eva/seal/seal.cpp:124-146
  Valuation decrypt(const B200Valuation &enc, const CKKSSignature &sig) {
    Valuation out;
    const u64 N = s_->dev->N();
    auto &encoder = s_->client->encoder();
    for (auto &e : enc) {
      if (auto *c = std::get_if<HostCipher>(&e.second)) {
        DBuf ct(s_->dev, c->data.size());
        s_->dev->upload(ct.get(), c->data.data(), c->data.size() * 8);
        DBuf pt = s_->client->decrypt(s_->keys, ct.get(), c->size, c->ell);
        out[e.first] = encoder.decode(pt.get(), c->ell, c->scale);
      } else if (auto *sc = std::get_if<HostSeededCipher>(&e.second)) {
        // c1 expanded from the seed on the device, then decrypted as a full ciphertext
        if (sc->ell < 1 || sc->ell > s_->dev->k() - 1 || sc->c0.size() != (std::size_t)sc->ell * N)
          throw std::runtime_error("value " + e.first + ": seeded ciphertext does not match the parameters (level / degree)");
        DBuf ct(s_->dev, 2 * sc->c0.size());
        s_->dev->upload(ct.get(), sc->c0.data(), sc->c0.size() * 8);
        u64 *c1 = ct.get() + sc->c0.size();
        expandCiphers(*s_->dev, 1, &sc->seed, &c1, &sc->ell, nullptr);
        DBuf pt = s_->client->decrypt(s_->keys, ct.get(), 2, sc->ell);
        out[e.first] = encoder.decode(pt.get(), sc->ell, sc->scale);
      } else if (auto *p = std::get_if<HostPlain>(&e.second)) {
        DBuf pt(s_->dev, (std::size_t)p->ell * N);
        s_->dev->upload(pt.get(), p->data.data(), (std::size_t)p->ell * N * 8);
        out[e.first] = encoder.decode(pt.get(), p->ell, p->scale);
      } else if (auto *r = std::get_if<StoredCipher>(&e.second)) {
        throw std::invalid_argument("value " + e.first + " is a reference to a stored ciphertext (handle " + std::to_string(r->handle) +
                                    "): only a server's requests can name one");
      } else if (auto *cc = std::get_if<HostCompactCipher>(&e.second)) {
        out[e.first] = decryptCompact(*cc, e.first, nullptr);
      } else {
        std::get<std::shared_ptr<ConstantValue>>(e.second)->expandTo(out[e.first], sig.vecSize);
      }
      out.at(e.first).resize(sig.vecSize);
    }
    return out;
  }
  // a compact response: z = (y0 + y1 s) mod 2^bits, centred, decoded at the compact scale.  y1 s is exact in RNS over the fewest
  // primes whose bit lengths sum to at least bits + 2 + log2 N (their product exceeds 2 (N+1) 2^bits); z is decoded over the fewest
  // whose bit lengths sum to at least bits + 1.  z (if not null) receives the N centred integers
  std::vector<double> decryptCompact(const HostCompactCipher &c, const std::string &name, std::vector<std::int64_t> *z) {
    if (!s_->keys.sk) throw std::runtime_error("this context has no secret key");
    const u64 N = s_->dev->N();
    const auto &primes = s_->dev->primes();
    const int k = s_->dev->k();
    if (c.bits < 1 || c.bits > 62) throw std::invalid_argument("value " + name + ": compact ciphertext bits must be in [1, 62]");
    const std::size_t W = (N * c.bits + 63) / 64;
    if (c.words.size() != 2 * W) throw std::invalid_argument("value " + name + ": compact ciphertext does not match the parameters (2 x W words)");
    auto fewest = [&](int need) {
      int have = 0;
      for (int i = 0; i < k && i < kCompactMaxEll; i++) { have += 63 - __builtin_clzll(primes[i]); if (have >= need) return i + 1; }
      throw std::runtime_error("value " + name + ": the modulus chain is too short to decrypt a " + std::to_string(c.bits) + "-bit compact ciphertext");
    };
    const int logN = 63 - __builtin_clzll(N);
    const int L = fewest(c.bits + 2 + logN), L2 = fewest(c.bits + 1);
    evab_ctx *ctx = s_->dev->ctx();
    std::vector<int> idx(std::max(L, L2));
    for (std::size_t i = 0; i < idx.size(); i++) idx[i] = (int)i;
    DBuf w(s_->dev, 2 * W), y(s_->dev, 2 * (std::size_t)L * N), t(s_->dev, (std::size_t)L * N), pt(s_->dev, (std::size_t)L2 * N), zd(s_->dev, N);
    s_->dev->upload(w.get(), c.words.data(), 2 * W * 8);
    check(evab_compact_unpack(ctx, w.get(), c.bits, L, y.get(), nullptr));
    check(evab_ntt_fwd(ctx, y.get(), 2 * (std::size_t)L, idx.data(), L, nullptr));
    check(evab_mul_plain(ctx, L, t.get(), y.get() + (std::size_t)L * N, 1, s_->keys.sk.get(), nullptr));
    check(evab_add(ctx, L, t.get(), t.get(), 1, y.get(), 1, nullptr));
    check(evab_ntt_inv(ctx, t.get(), (std::size_t)L, idx.data(), L, nullptr));
    check(evab_compact_finish(ctx, t.get(), L, c.bits, L2, pt.get(), reinterpret_cast<std::int64_t *>(zd.get()), nullptr));
    if (z) {
      z->resize(N);
      s_->dev->download(z->data(), zd.get(), N * 8);
    }
    check(evab_ntt_fwd(ctx, pt.get(), (std::size_t)L2, idx.data(), L2, nullptr));
    s_->dev->sync();
    return s_->client->encoder().decode(pt.get(), L2, c.scale);
  }
  std::shared_ptr<Shared> shared() const { return s_; }
private:
  std::shared_ptr<Shared> s_;
};

// generateKeys -- reference eva/seal/seal.cpp:174-203
inline std::tuple<std::unique_ptr<B200Public>, std::unique_ptr<B200Secret>>
generateKeys(const CKKSParameters &params, int device = 0, std::uint64_t seed = 0, const std::string &rotationKeys = "program") {
  const std::vector<int> rots = rotationKeySteps(params, rotationKeys);
  std::vector<int> bits(params.primeBits.begin(), params.primeBits.end());
  auto primes = hmod::createCoeffModulus(params.polyModulusDegree, bits);
  auto s = std::make_shared<Shared>();
  s->dev = std::make_shared<Device>(params.polyModulusDegree, primes, device);
  // seed == 0 (the default): keys and encryption randomness from a CSPRNG keyed with 256 bits of OS entropy;
  // a non-zero seed is the deterministic test path (host/csprng.hpp)
  s->client = std::make_unique<CkksClient>(s->dev, seed);
  s->client->keygen(s->keys, rots);
  return std::make_tuple(std::make_unique<B200Public>(s), std::make_unique<B200Secret>(s));
}

}  // namespace evab
