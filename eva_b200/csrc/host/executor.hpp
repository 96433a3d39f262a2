// executor.hpp -- GPU executor + stream/graph DAG scheduler for compiled EVA
// programs.  Replaces, for the hot path,
//   SEALExecutor::operator()/setInputs/getOutputs/free  (reference eva/seal/seal_executor.h:264-436)
//   ProgramTraversal / MulticoreProgramTraversal::forwardPass
//                                                       (eva/common/program_traversal.h:36-88,
//                                                        eva/common/multicore_program_traversal.h:24-84)
// Instead of interpreting the DAG term by term on CPU threads, the program is
// lowered ONCE into a static plan (planner.hpp: value kinds, levels, scales, device buffer
// offsets, stream assignment, event edges); every execute() then replays the
// plan: independent terms run concurrently on different CUDA streams, cross-
// stream dependencies are events, and the whole replay can be captured into a
// CUDA graph so that one execute() costs a single graph launch.
#pragma once
#include "ckks_client.hpp"
#include "logging.hpp"
#include "planner.hpp"
#include <nvtx3/nvToolsExt.h>
#include <unordered_set>

namespace evab {

// scoped evab_set_batch: ops issued by this thread act on `batch` instances
struct BatchGuard {
  BatchGuard(int batch, std::size_t stride, std::size_t vstride) { check(evab_set_batch(batch, stride, vstride)); }
  ~BatchGuard() { evab_set_batch(1, 0, 0); }
};
// scoped evab_set_key_bank: batch instance b of the ops issued by this thread reads the keys of tenant d_tenant[b] (null: shared keys)
struct KeyBankGuard {
  KeyBankGuard(const std::int32_t *d_tenant, std::size_t stride) { check(evab_set_key_bank(d_tenant, stride)); }
  ~KeyBankGuard() { evab_set_key_bank(nullptr, 0); }
};
// scoped evab_set_hoist_inline: the hoisted rotations issued by this thread read indicator rows as their constants
struct HoistInlineGuard {
  explicit HoistInlineGuard(bool on) { check(evab_set_hoist_inline(on ? 1 : 0)); }
  ~HoistInlineGuard() { evab_set_hoist_inline(0); }
};
// scoped evab_set_key_seeded: the key switches issued by this thread read seeded key images and draw their c1 words
struct KeySeededGuard {
  explicit KeySeededGuard(bool on) { check(evab_set_key_seeded(on ? 1 : 0)); }
  ~KeySeededGuard() { evab_set_key_seeded(0); }
};
// scoped evab_set_key_c1_rows: batch instance b of the key switches issued by this thread reads cached c1 rows from region
// d_region[b] of the key bank, or draws them (-1); null: every instance draws
struct KeyC1Guard {
  explicit KeyC1Guard(const std::int32_t *d_region) { check(evab_set_key_c1_rows(d_region)); }
  ~KeyC1Guard() { evab_set_key_c1_rows(nullptr); }
};

// Evaluation keys of up to `capacity` tenants (one client's key set each) in one device allocation.  Every tenant's region has
// the same layout -- the relinearization key, one Galois key per element of the rotation set, then the hoist constants cadd of
// every (element, ell) with ell = 1 .. k-1 (one evab_rotate_hoist_const_levels call, when the region is filled) -- so region t's
// copy of any of them is at region 0's pointer + t * stride() words.  Plans take region 0's pointers and select per instance at
// run time.  Without paging a tenant id is its region; with paging (KeyPager) the regions are slots that tenants are paged into.
// Inline hoist constants (inlineConstants): a region holds the keys only, and the bank one copy of every element's indicator rows
// NTT_m(I_g) [k][N], shared by all tenants; the hoisted rotations form each constant from those rows and the keys they load
// (evab_set_hoist_inline), so fills compute nothing.
// Seeded keys (seededKeys, inline constants only): every key of a region is a self-contained seeded image -- its c0 rows [k-1][k][N],
// then its 32-byte seed padded to 64 bytes (evab_seeded_key_bytes) -- and the key switches draw the c1 rows from the seed
// (evab_set_key_seeded).  The compressed host image of a tenant is the region's own layout, so a fill is one upload and no launch.
// c1 regions (c1Regions, seeded keys only): the allocation continues with that many regions of the same stride after the capacity
// slots; region capacity + h holds the expanded c1 rows of one tenant's keys, key i's rows [k-1][k][N] at the word offset of its c0
// rows in a seeded image (fillC1, evab_expand_seeded_c1), and an instance whose c1 table entry is capacity + h reads them
// (evab_set_key_c1_rows) instead of drawing them.
class KeyBank {
public:
  KeyBank(std::shared_ptr<Device> dev, const std::set<u64> &elts, int capacity, bool inlineConstants = false, bool seededKeys = false,
          int c1Regions = 0)
      : dev_(std::move(dev)), elts_(elts.begin(), elts.end()), inline_(inlineConstants), seeded_(seededKeys), c1Regions_(c1Regions) {
    if (capacity < 1 || capacity > 65535) throw std::invalid_argument("key bank capacity must be in [1, 65535]");
    if (seeded_ && !inline_) throw std::invalid_argument("a bank of seeded keys forms its hoist constants inline");
    if (c1Regions_ < 0 || c1Regions_ > capacity || (c1Regions_ && !seeded_))
      throw std::invalid_argument("c1 regions: 0 .. capacity, and only in a bank of seeded keys");
    const std::size_t N = dev_->N(), k = (std::size_t)dev_->k();
    if (k < 2) throw std::invalid_argument("a key bank needs at least two primes");
    keyWords_ = seeded_ ? evab_seeded_key_bytes(dev_->ctx()) / 8 : (k - 1) * 2 * k * N;
    if (!inline_)
      for (std::size_t ell = 1; ell < k; ell++) constWords_ += 2 * (ell + 1) * N;
    stride_ = keyWords_ * (1 + elts_.size()) + constWords_ * elts_.size();
    for (u64 e : elts_) check(evab_galois_prepare(dev_->ctx(), e));
    bank_ = DBuf(dev_, stride_ * ((std::size_t)capacity + (std::size_t)c1Regions_));
    if (!seeded_) seeds_ = DBuf(dev_, 4 * keys() * (std::size_t)capacity);
    if (!elts_.empty() && !inline_) tmp_ = DBuf(dev_, evab_rotate_hoist_const_levels_work_bytes(dev_->ctx(), (int)elts_.size()) / 8);
    if (!elts_.empty() && inline_) {
      ind_ = DBuf(dev_, evab_hoist_indicators_bytes(dev_->ctx(), (int)elts_.size()) / 8);
      check(evab_hoist_indicators(dev_->ctx(), (int)elts_.size(), elts_.data(), ind_.get(), nullptr));
    }
    used_.assign(capacity, 0);
    dev_->sync();
  }
  bool inlineConstants() const { return inline_; }
  bool seededKeys() const { return seeded_; }
  int c1Regions() const { return c1Regions_; }
  // the c1 rows of every key of the tenant in slot `slot` -> c1 region h (one launch, stream-ordered; the slot's images must be there)
  void fillC1(int h, int slot, void *stream) {
    if (h < 0 || h >= c1Regions_) throw std::logic_error("c1 region out of range");
    check(evab_expand_seeded_c1(dev_->ctx(), (int)keys(), region(slot), region(capacity() + h), stream));
  }  // the indicator rows [k][N] of an element (inline constants; one copy for every tenant)
  const u64 *indicators(u64 elt) const {
    if (!inline_) throw std::logic_error("indicator rows are kept by banks with inline hoist constants only");
    return ind_.get() + index(elt) * (std::size_t)dev_->k() * dev_->N();
  }
  std::size_t indicatorBytes() const { return inline_ ? elts_.size() * (std::size_t)dev_->k() * dev_->N() * 8 : 0; }
  int capacity() const { return (int)used_.size(); }
  int tenants() const { return (int)std::count_if(used_.begin(), used_.end(), [](char u) { return u != 0; }); }
  int compressedTenants() const { return (int)std::count(used_.begin(), used_.end(), 2); }
  std::size_t stride() const { return stride_; }                 // words
  std::size_t keys() const { return 1 + elts_.size(); }            // the relinearization key, then a Galois key per element
  std::size_t keyWords() const { return keyWords_ * keys(); }
  // a compressed tenant's host image: the c0 rows [k-1][k][N] of every key (in region order), then the keys' 32-byte seeds; seeded
  // keys: the region's keys (seeded images)
  std::size_t compressedWords() const { return seeded_ ? keyWords() : keyWords() / 2 + 4 * keys(); }
  std::size_t constWords() const { return constWords_ * elts_.size(); }
  const std::vector<u64> &elements() const { return elts_; }
  bool has(u64 elt) const { return std::binary_search(elts_.begin(), elts_.end(), elt); }
  bool occupied(int t) const { return t >= 0 && t < capacity() && used_[t]; }
  void requireOccupied(int t) const {
    if (!occupied(t)) throw std::invalid_argument("tenant " + std::to_string(t) + " has no keys on this server");
  }
  // tenant 0's copies (the layout shared by every tenant)
  const u64 *relin(int t = 0) const { return bank_.get() + (std::size_t)t * stride_; }
  const u64 *galois(u64 elt, int t = 0) const { return relin(t) + keyWords_ * (1 + index(elt)); }
  const u64 *hoistConst(u64 elt, int ell, int t = 0) const {
    if (inline_) throw std::logic_error("a bank with inline hoist constants stores none");
    if (ell < 1 || ell >= dev_->k()) throw std::invalid_argument("hoist constant level out of range");
    std::size_t off = keyWords_ * (1 + elts_.size()) + constWords_ * index(elt);
    for (int l = 1; l < ell; l++) off += 2 * (std::size_t)(l + 1) * dev_->N();
    return relin(t) + off;
  }
  // copies host images [k-1][2][k][N] (shapes checked by the caller) of the relinearization key and of a Galois key for every
  // element into a free region and computes its hoist constants (stored constants only); returns the tenant id
  int add(const u64 *relinKey, const std::map<u64, const u64 *> &galoisKeys) {
    if (seeded_) throw std::logic_error("a bank of seeded keys takes compressed keys only");
    const auto it = std::find(used_.begin(), used_.end(), 0);
    if (it == used_.end()) throw std::runtime_error("the key bank is full (" + std::to_string(capacity()) + " tenants): remove a tenant first");
    const int t = (int)(it - used_.begin());
    dev_->upload(region(t), relinKey, keyWords_ * 8);
    for (u64 e : elts_) dev_->upload(const_cast<u64 *>(galois(e, t)), galoisKeys.at(e), keyWords_ * 8);
    computeConstants(t, nullptr);
    dev_->sync();
    used_[t] = 1;
    return t;
  }
  // the same from a compressed image (compressedWords() words, packed by packCompressed): the c0 rows are uploaded, the c1 rows
  // expanded from the seeds on the device
  int addCompressed(const u64 *image) {
    const auto it = std::find(used_.begin(), used_.end(), 0);
    if (it == used_.end()) throw std::runtime_error("the key bank is full (" + std::to_string(capacity()) + " tenants): remove a tenant first");
    const int t = (int)(it - used_.begin());
    fillCompressed(t, image, nullptr);
    dev_->sync();
    *it = 2;
    return t;
  }
  // host images [k-1][k][N] of the c0 rows and the seeds of the relinearization key and every element's Galois key -> dst
  void packCompressed(u64 *dst, const u64 *relinC0, const KeySeed &relinSeed, const std::map<u64, std::pair<const u64 *, KeySeed>> &galois) const {
    if (seeded_) {   // key i: c0 rows then the seed, at i keyWords_
      const std::size_t w = keyWords_ - 8;
      auto put = [&](std::size_t i, const u64 *c0, const KeySeed &seed) {
        std::memcpy(dst + i * keyWords_, c0, w * 8);
        std::memset(dst + i * keyWords_ + w, 0, 64);
        std::memcpy(dst + i * keyWords_ + w, seed.data(), 32);
      };
      put(0, relinC0, relinSeed);
      for (std::size_t i = 0; i < elts_.size(); i++) put(1 + i, galois.at(elts_[i]).first, galois.at(elts_[i]).second);
      return;
    }
    const std::size_t w = keyWords_ / 2;
    std::memcpy(dst, relinC0, w * 8);
    std::memcpy(dst + keys() * w, relinSeed.data(), 32);
    for (std::size_t i = 0; i < elts_.size(); i++) {
      const auto &g = galois.at(elts_[i]);
      std::memcpy(dst + (1 + i) * w, g.first, w * 8);
      std::memcpy(dst + keys() * w + 4 * (1 + i), g.second.data(), 32);
    }
  }
  void remove(int t) { requireOccupied(t); used_[t] = 0; }
  // paging (B200Server with more tenants than regions): region `slot` takes the keys of a host block laid out as a region's keys
  // ([relinearization key][Galois key of every element], keyWords() words) and recomputes the constants; stream-ordered, no sync
  void fill(int slot, const u64 *hostKeys, void *stream) {
    dev_->upload(region(slot), hostKeys, keyWords() * 8, stream);
    computeConstants(slot, stream);
  }
  // the same from a compressed image: one strided upload puts every c0 row in its place (the digits of all keys are (k-1) keys()
  // rows of k N words, 2 k N words apart in the region), the seeds go to the slot's seed block, one launch expands every c1 row
  // (seeded keys: the image is the region's keys, one upload)
  void fillCompressed(int slot, const u64 *image, void *stream) {
    if (seeded_) {
      dev_->upload(region(slot), image, keyWords() * 8, stream);
      computeConstants(slot, stream);   // counts the fill; inline constants compute nothing
      return;
    }
    const std::size_t kN = (std::size_t)dev_->k() * dev_->N(), rows = keys() * ((std::size_t)dev_->k() - 1);
    check(evab_upload_2d(dev_->ctx(), region(slot), 2 * kN * 8, image, kN * 8, kN * 8, rows, stream));
    u64 *seeds = seeds_.get() + 4 * keys() * (std::size_t)slot;
    dev_->upload(seeds, image + rows * kN, 32 * keys(), stream);
    expandKeys(*dev_, (int)keys(), seeds, region(slot), stream);
    computeConstants(slot, stream);
  }
  // the hoist constants of every (element, ell) of region `slot` from its Galois keys (one evab_rotate_hoist_const_levels call:
  // the region's Galois keys and constants are each contiguous, in element order); inline constants: nothing to compute
  void computeConstants(int slot, void *stream) {
    fills_++;
    if (elts_.empty() || inline_) return;
    check(evab_rotate_hoist_const_levels(dev_->ctx(), (int)elts_.size(), elts_.data(), galois(elts_[0], slot), const_cast<u64 *>(hoistConst(elts_[0], 1, slot)),
                                         tmp_.get(), stream));
  }
  std::uint64_t fills() const { return fills_; }

private:
  std::size_t index(u64 elt) const {
    auto it = std::lower_bound(elts_.begin(), elts_.end(), elt);
    if (it == elts_.end() || *it != elt) throw std::invalid_argument("Galois key not present");
    return (std::size_t)(it - elts_.begin());
  }
  u64 *region(int t) const { return bank_.get() + (std::size_t)t * stride_; }
  std::shared_ptr<Device> dev_;
  std::vector<u64> elts_;                 // sorted
  bool inline_ = false;                   // inline hoist constants: no constants in the regions, ind_ holds the indicator rows
  bool seeded_ = false;                   // seeded keys: keyWords_ is one seeded image, no seeds_ (the seeds are in the images)
  int c1Regions_ = 0;                     // c1 regions after the capacity slots (seeded keys)
  std::size_t keyWords_ = 0, constWords_ = 0, stride_ = 0;   // one key; the constants of one element; one tenant
  std::vector<char> used_;                // 0: free, 1: keys added in full, 2: added compressed
  std::uint64_t fills_ = 0;               // regions filled (keys uploaded, constants computed)
  DBuf bank_, tmp_, seeds_;               // seeds_: [region][keys()][32 bytes], the seeds of the region's last compressed fill                       // tmp_: the indicators of computeConstants (fills are ordered on one stream at a time)
  DBuf ind_;                              // inline constants: [element][k][N] NTT_m(I_g)
};

class Executor {
public:
  // bank != null: keys come from the bank, tenant per instance (setKeyTable); `keys` is not read.  The plan is the same either way.
  Executor(std::shared_ptr<Device> dev, const KeySet &keys, Program &program, ExecOptions opt = {}, const KeyBank *bank = nullptr)
      : dev_(std::move(dev)), keys_(keys), bank_(bank), prog_(program), plan_(plan(opt)), N_(dev_->N()) {
    materialise();
  }
  ~Executor() {
    if (graph_) evab_graph_destroy(dev_->ctx(), graph_);
    if (hostFlags_) evab_host_free(hostFlags_);
    if (keyTableHost_) evab_host_free(keyTableHost_);
    for (void *e : events_) evab_event_destroy(dev_->ctx(), e);
    for (void *s : streams_) evab_stream_destroy(dev_->ctx(), s);
  }
  Executor(const Executor &) = delete;

  std::size_t cipherOpCount() const { return plan_.cipherOps; }
  // shape of the plan (test / tooling hook)
  std::map<std::string, long> planStats() const { return plan_.planStats(); }
  // false when the plan's arena is packed and the value's storage may have been reused by a later value of the run
  bool intact(std::uint64_t index) const { const int r = plan_.storage.at(index); return !plan_.packed || (r >= 0 && plan_.regions[r].pinned); }
  std::size_t arenaBytes() const { return plan_.arenaBytes(); }
  // private stream used by B200Public::execute for H2D -> run -> D2H of this plan,
  // so that execute() calls on different programs overlap on the GPU
  void *mainStream() {
    if (!mainStream_) { check(evab_stream_create(dev_->ctx(), &mainStream_)); streams_.push_back(mainStream_); }
    return mainStream_;
  }
  const ValueInfo &info(const Term::Ptr &t) const { return plan_.vals.at(t->index); }
  int batch() const { return plan_.opt.batch; }
  u64 *valuePtr(const Term::Ptr &t, int b = 0) const { return valuePtr(t->index, b); }
  u64 *valuePtr(std::uint64_t index, int b = 0) const { return arena_.get() + (std::size_t)b * plan_.stride + plan_.vals.at(index).off; }
  const ValueInfo &info(std::uint64_t index) const { return plan_.vals.at(index); }
  const std::vector<double> &rawValue(std::uint64_t index, int b = 0) const { return rawsB_.at(b).at(index); }

  // device-resident run: inputs must already be in valuePtr(input term); raw
  // inputs set through setRawInput.  Enqueues the whole program on `stream`
  // (graph launch or multi-stream replay); does not synchronise.
  // the key table of the next runs (bank-bound executors): the bank slot of every instance, then, for a bank with c1 regions, its
  // c1 table entry, capacity + h or -1 (draws); c1 is null exactly when the bank has no c1 regions.  The page-locked copy is read
  // by run()'s stream-ordered upload: callers rewrite it only once the previous run's stream has been synchronised
  void setKeyTable(const int *slots, const int *c1, int n) {
    if (!bank_ || n != plan_.opt.batch || !c1 != !c1Table())
      throw std::logic_error("setKeyTable: one slot per instance of a bank-bound plan, and c1 entries exactly when the bank has c1 regions");
    std::copy(slots, slots + n, keyTableHost_);
    if (c1) std::copy(c1, c1 + n, keyTableHost_ + n);
  }
  bool keyTableIs(const int *slots, const int *c1, int n) const {
    return bank_ && n == plan_.opt.batch && !c1 == !c1Table() && std::equal(slots, slots + n, keyTableHost_) &&
           (!c1 || std::equal(c1, c1 + n, keyTableHost_ + n));
  }
  void run(void *stream) {
    if (rawDirty_) { evalRawAndEncodes(stream); rawDirty_ = false; }
    if (bank_) dev_->upload(keyTableDev_.get(), keyTableHost_, 4 * keyTableEntries(), stream);   // read by the kernels, not baked into the graph
    if (plan_.opt.useGraph && verbosity() < 2) {   // debug verbosity: step-by-step replay so that every term is reported
      if (!graph_ || !graphValid_) capture();
      check(evab_graph_launch(dev_->ctx(), graph_, stream));
    } else {
      replay(stream);
    }
    for (int b = 0; plan_.numFlags && b < plan_.opt.batch; b++)   // travels with the outputs; read by flagsRaised() once the stream is synchronised
      dev_->download(hostFlags_ + (std::size_t)b * 8 * plan_.numFlags, arena_.get() + (std::size_t)b * plan_.stride + plan_.flagsOff,
                     8 * plan_.numFlags * 8, stream);
  }
  // after the run's stream has been synchronised: did a digit of a rotation group hold a zero coefficient?  (The shared mod-up is
  // then not the reference's value; the caller must redo the run with hoistModUp off.  Probability ~ N ell 2^-60 per ciphertext.)
  bool flagsRaised() const {
    for (std::size_t i = 0; i < 8 * plan_.numFlags * (std::size_t)plan_.opt.batch; i++)
      if (hostFlags_[i]) return true;
    return false;
  }
  void setRawInput(const std::string &name, const std::vector<double> &v, int b = 0) {
    auto t = prog_.getInput(name);
    if (plan_.vals.at(t->index).kind != Kind::Raw) throw std::runtime_error("input " + name + " is not a raw input");
    std::vector<double> x;
    ConstantValue(prog_.getVecSize(), v).expandTo(x, prog_.getVecSize());
    rawsB_.at(b)[t->index] = x;
    rawDirty_ = true;
  }

private:
  // ---------------------------------------------------------------- planning
  Plan plan(const ExecOptions &opt) const {
    const evab_ctx *c = dev_->ctx();
    WorkSizes ws;
    ws.keyswitch = [c](int ell) { return evab_keyswitch_work_bytes(c, ell); };
    ws.rotateModupExt = [c](int ell) { return evab_rotate_modup_ext_bytes(c, ell); };
    ws.rescale = [c](int size) { return evab_rescale_work_bytes(c, size); };
    ws.rotateModupMany = [c](int ell, int n) { return evab_rotate_modup_many_work_bytes(c, ell, n); };
    ws.rotateWsum = [c](int ell, int n, int nout) { return evab_rotate_wsum_work_bytes(c, ell, n, nout); };
    ws.lazyRotsum = [c](int ell, int nout) { return evab_lazy_rotsum_work_bytes(c, ell, nout); };
    ws.encode = [c](int count) { return evab_encode_work_bytes(c, count); };
    if (bank_ && bank_->inlineConstants() && opt.approxHoist)
      throw std::invalid_argument("approx_hoist needs stored hoist constants: this server was built with hoist_constants=\"inline\"");
    std::size_t limit = opt.arenaLimit;
    if (!limit) { std::size_t freeB = 0, totalB = 0; check(evab_mem_info(dev_->ctx(), &freeB, &totalB)); limit = freeB; }
    std::set<u64> elts;   // rotations by steps without a key of their own are composed (planner.hpp composeRotations)
    if (bank_) elts.insert(bank_->elements().begin(), bank_->elements().end());
    else for (auto &g : keys_.galois) elts.insert(g.first);
    return buildPlan(prog_, opt, dev_->N(), dev_->k(), limit, ws, &elts);
  }
  // device side of the plan: arenas, streams, events, plan-time encodes, Galois tables and hoist constants
  void materialise() {
    const Plan &p = plan_;
    const int B = p.opt.batch;
    rawsB_.assign(B, p.constants);
    arena_ = DBuf(dev_, p.stride * B + 8);
    rawArena_ = DBuf(dev_, p.rawStride * B + 8);
    dev_->sync();  // stream-ordered allocation made on the null stream: publish it to the plan's streams
    for (int s = 0; s < p.usedStreams; s++) { void *h; check(evab_stream_create(dev_->ctx(), &h)); streams_.push_back(h); }
    for (int e = 0; e < p.numEvents + p.usedStreams + 1; e++) { void *h; check(evab_event_create(dev_->ctx(), &h)); events_.push_back(h); }
    // plan-time constants: raw values and (optionally) their encodings
    evalRawAndEncodes(nullptr);
    rawDirty_ = false;
    // Galois tables of every rotation; for each (element, ell) a shared mod-up serves, its key-dependent constant (a key bank
    // holds those of every tenant)
    std::set<std::pair<u64, int>> done;   // ell 0: Galois table only
    p.forEachRotation([&](const Term *r, bool hoisted) {
      const u64 elt = galoisElt(*r);
      if (!(bank_ ? bank_->has(elt) : keys_.galois.count(elt) > 0)) throw std::invalid_argument("Galois key not present");
      const int ell = hoisted ? p.vals[r->index].ell : 0;
      if (!done.emplace(elt, ell).second) return;
      check(evab_galois_prepare(dev_->ctx(), elt));
      if (!ell || bank_) return;
      DBuf cadd(dev_, evab_hoist_const_bytes(dev_->ctx(), ell) / 8), tmp(dev_, (std::size_t)(ell + 1) * N_);
      check(evab_rotate_hoist_const(dev_->ctx(), ell, elt, keys_.galois.at(elt).get(), cadd.get(), tmp.get(), nullptr));
      dev_->sync();
      hoistConst_.emplace(std::make_pair(elt, ell), std::move(cadd));
    });
    if (p.numFlags) check(evab_host_alloc(8 * p.numFlags * 8 * (std::size_t)B, (void **)&hostFlags_));
    if (bank_) {
      keyTableDev_ = DBuf(dev_, (keyTableEntries() + 1) / 2);
      check(evab_host_alloc(4 * keyTableEntries(), (void **)&keyTableHost_));
      std::fill(keyTableHost_, keyTableHost_ + B, 0);
      std::fill(keyTableHost_ + B, keyTableHost_ + keyTableEntries(), -1);
      dev_->sync();
    }
  }
  bool c1Table() const { return bank_ && bank_->c1Regions() > 0; }
  std::size_t keyTableEntries() const { return (std::size_t)plan_.opt.batch * (c1Table() ? 2 : 1); }
  const u64 *relinKey() const { return bank_ ? bank_->relin() : keys_.relin.get(); }
  const u64 *galoisKey(u64 elt) const { return bank_ ? bank_->galois(elt) : keys_.galois.at(elt).get(); }
  // a hoisted rotation's constant operand: cadd_g at level ell, or with inline constants the element's indicator rows
  const u64 *hoistConst(u64 elt, int ell) const {
    if (bank_) return bank_->inlineConstants() ? bank_->indicators(elt) : bank_->hoistConst(elt, ell);
    return hoistConst_.at(std::make_pair(elt, ell)).get();
  }
  // the element of the rotation a term applies (a hop of a composed rotation: its term's)
  u64 galoisElt(const Term &t) const {
    const u64 elt = evab_galois_elt_from_step(N_, plan_.stepOf(&t));
    if (!elt) throw std::invalid_argument("step count too large");
    return elt;
  }

  // raw (vector<double>) terms run on the host (reference seal_executor.h:63-112);
  // Encode terms whose operand does not depend on raw inputs are encoded once.
  void evalRawAndEncodes(void *stream) {
    const Plan &p = plan_;
    for (int b = 0; b < p.opt.batch; b++) {
      auto &raws = rawsB_[b];
      for (auto &t : p.order) {
        const ValueInfo &v = p.vals[t->index];
        if (v.kind == Kind::Raw && t->op != Op::Input && t->op != Op::Constant) {
          auto &out = raws[t->index];
          auto &x = raws[t->operandAt(0)->index];
          if (t->op == Op::Output) { out = x; continue; }
          if (x.empty()) { out.clear(); continue; }  // raw input not provided yet
          const std::size_t n = x.size();
          out.resize(n);
          if (t->op == Op::Negate) for (std::size_t i = 0; i < n; i++) out[i] = -x[i];
          else if (t->op == Op::RotateLeftConst || t->op == Op::RotateRightConst) {
            long long sh = *t->rotation;
            if (t->op == Op::RotateRightConst) sh = -sh;
            sh %= (long long)n; if (sh < 0) sh += n;
            for (std::size_t i = 0; i < n; i++) out[i] = x[(i + sh) % n];
          } else {
            auto &y = raws[t->operandAt(1)->index];
            if (y.empty()) { out.clear(); continue; }
            for (std::size_t i = 0; i < n; i++) out[i] = t->op == Op::Add ? x[i] + y[i] : t->op == Op::Sub ? x[i] - y[i] : x[i] * y[i];
          }
        }
        if (t->op == Op::Encode) {
          if (p.encodeAlias.count(t->index)) continue;
          auto &x = raws[t->operandAt(0)->index];
          if (x.empty()) continue;
          const std::uint64_t key = t->index * 65536ull + (std::uint64_t)b;
          if (!rawUploaded_.count(key) || p.dyn[t->index]) {
            if ((N_ / 2) % x.size()) throw std::runtime_error("Vector size must exactly divide the slot count");
            dev_->upload(rawArena_.get() + (std::size_t)b * p.rawStride + p.rawOff.at(t->index), x.data(), x.size() * 8, stream);
            rawUploaded_.insert(key);
          }
        }
      }
    }
    dev_->sync(stream);  // the staged host vectors must outlive the copies
    if (p.opt.cacheConstants && !staticEncoded_) {
      BatchGuard bg(p.opt.batch, p.stride, p.rawStride);
      for (auto &g : p.groups) if (!g.dynamic) issueEncodeGroup(g, stream);
      dev_->sync(stream);
      staticEncoded_ = true;
    }
  }
  // one batched device encode (scatter -> inverse FFT -> round/reduce -> NTT) for a group
  void issueEncodeGroup(const EncodeGroup &g, void *stream) {
    if (g.nUniform) {   // replicated scalars: constant polynomials, no FFT / NTT needed (bit-identical)
      std::vector<double> v, sc;
      for (int i = 0; i < g.nUniform; i++) { v.push_back(rawsB_[0][g.members[i]->operandAt(0)->index][0]); sc.push_back(plan_.vals[g.members[i]->index].scale); }
      check(evab_encode_uniform_ext(dev_->ctx(), g.nUniform, v.data(), sc.data(), g.ell, g.withP ? 1 : 0, arena_.get() + g.outOff, stream));
    }
    const int rest = (int)g.members.size() - g.nUniform;
    if (!rest) return;
    std::vector<const double *> ptrs; std::vector<std::uint32_t> vec; std::vector<double> sc;
    for (int i = g.nUniform; i < (int)g.members.size(); i++) {
      Term *t = g.members[i];
      ptrs.push_back(reinterpret_cast<const double *>(rawArena_.get() + plan_.rawOff.at(t->index)));
      vec.push_back((std::uint32_t)rawsB_[0][t->operandAt(0)->index].size());
      sc.push_back(plan_.vals[t->index].scale);
    }
    check(evab_encode_ext(dev_->ctx(), rest, ptrs.data(), vec.data(), sc.data(), g.ell, g.withP ? 1 : 0,
                          arena_.get() + g.outOff + (std::size_t)g.nUniform * (g.ell + (g.withP ? 1 : 0)) * N_, arena_.get() + g.workOff, stream));
  }
  // ---------------------------------------------------------------- execution
  // Tracing (reference eva/seal/seal_executor.h:280-294 prints every term at EVA_VERBOSITY >= debug; SURVEY section 5
  // asks for NVTX ranges): with EVA_VERBOSITY=debug the plan is replayed step by step (no CUDA graph) and every
  // step prints the reference's line -- followed by the stream it was issued on -- and is wrapped in an NVTX range
  // named after its term, so that nsys / ncu timelines read in program terms.  EVAB_NVTX=1 gives the ranges alone.
  struct TraceScope {
    bool nvtx;
    TraceScope(const Plan &p, const Step &st, bool print, bool nvtx_) : nvtx(nvtx_) {
      if (!print && !nvtx) return;
      char name[96];
      const Term &t = *st.term;
      const bool term = st.kind == StepKind::Term;
      const char *pseudo = st.kind == StepKind::RotationChunk ? "RotationBatch" : st.kind == StepKind::RotationSum ? "LazyRotationSums" : "InverseNTT";
      if (!term) std::snprintf(name, sizeof(name), "t%lu.%s", (unsigned long)t.index, pseudo);
      else std::snprintf(name, sizeof(name), "t%lu %s%s", (unsigned long)t.index, opName(t.op), st.sum.empty() ? "" : "(fused sum)");
      if (print) {
        std::printf("EVA: Execute t%lu%s = %s(", (unsigned long)t.index, term ? "" : "'", term ? opName(t.op) : pseudo);
        bool first = true;
        if (!term) std::printf("t%lu", (unsigned long)t.index);
        else if (p.chainSrc.count(t.index)) std::printf("t%lu", (unsigned long)p.src(&t)->index);   // a hop of a composed rotation
        else for (auto &o : t.getOperands()) { std::printf(first ? "t%lu" : ",t%lu", (unsigned long)o->index); first = false; }
        std::printf(")  [stream %d%s]\n", st.stream, st.sum.empty() ? "" : ", fused sum");
        std::fflush(stdout);
      }
      if (nvtx) nvtxRangePushA(name);
    }
    ~TraceScope() { if (nvtx) nvtxRangePop(); }
  };
  static bool traceNvtx() { static const bool v = std::getenv("EVAB_NVTX") != nullptr || verbosity() >= 2; return v; }
  void issue(const Step &st, void *stream) {
    const Plan &p = plan_;
    const Term &t = *st.term;
    TraceScope trace(p, st, verbosity() >= 2, traceNvtx());
    evab_ctx *c = dev_->ctx();
    const ValueInfo &o = p.vals[t.index];
    u64 *const A = arena_.get();
    u64 *out = A + o.off;
    u64 *work = A + p.workOff[st.stream];
    std::vector<u64> elts; std::vector<const u64 *> keys, cadds;   // a chunk's or a rotation sum's rotations
    auto hoisted = [&](const std::vector<const Term *> &rots, int ell) {
      for (const Term *r : rots) {
        const u64 elt = galoisElt(*r);
        elts.push_back(elt); keys.push_back(galoisKey(elt));
        cadds.push_back(hoistConst(elt, ell));
      }
    };
    switch (st.kind) {
      case StepKind::RotationChunk: {   // up to 16 rotations of one ciphertext, three launches
        const RotChunk &ch = p.chunks[st.index];
        if (verbosity() >= 2)
          for (const Term *r : ch.rots)
            std::printf("EVA: Execute t%lu = %s(t%lu)  [stream %d, in the batch above]\n", (unsigned long)r->index, opName(r->op), (unsigned long)(p.chainSrc.count(r->index) ? p.src(r) : r->operandAt(0).get())->index, st.stream);
        hoisted(ch.rots, ch.ell);
        check(evab_rotate_modup_many(c, ch.ell, (int)elts.size(), A + ch.outOff, out, A + p.hoistExtOff[ch.gid], elts.data(), keys.data(), cadds.data(), work, stream));
        return;
      }
      case StepKind::RotationSum: {   // out_o = sum_i w_oi (.) rotate(x, g_i): approxHoist, one mod-down per sum; rotationSums, exact (+ taps)
        const LazySum &Lz = p.lazy[st.index];
        std::vector<const u64 *> wts, taps, twts;
        hoisted(Lz.rots, Lz.ell);
        for (auto &ws : Lz.wts) for (const Term *w : ws) wts.push_back(w ? A + p.vals[w->index].off : nullptr);
        if (!p.opt.approxHoist) {
          for (const Term *x : Lz.taps) taps.push_back(A + p.vals[x->index].off);
          for (auto &ws : Lz.twts) for (const Term *w : ws) twts.push_back(w ? A + p.vals[w->index].off : nullptr);
          check(evab_rotate_wsum(c, Lz.ell, (int)Lz.roots.size(), A + Lz.tempOff, out, A + p.hoistExtOff[Lz.gid], (int)elts.size(),
                                 elts.data(), keys.data(), cadds.data(), wts.data(), (int)taps.size(), taps.data(), twts.data(), work, stream));
          return;
        }
        check(evab_lazy_rotsum(c, Lz.ell, (int)Lz.roots.size(), A + Lz.tempOff, out, A + p.hoistExtOff[Lz.gid], (int)elts.size(),
                               elts.data(), keys.data(), cadds.data(), wts.data(), work, stream));
        return;
      }
      case StepKind::Hoist: {   // shared inverse NTT of a rotation group's input
        const int g = st.index;
        if (p.opt.hoistModUp) {
          check(evab_rotate_modup_prepare(c, o.ell, A + p.hoistOff[g], A + p.hoistExtOff[g], out, A + p.flagsOff + 8 * (std::size_t)g, stream));
          if (p.needsC0[g]) check(evab_rotate_modup_scale_c0(c, o.ell, A + p.hoistExtOff[g], out, stream));
        } else {
          check(evab_rotate_prepare(c, o.ell, A + p.hoistOff[g], out, stream));
        }
        return;
      }
      case StepKind::Term: break;
    }
    if (!st.sum.empty() || !st.rotSums.empty()) {   // fused multiply_plain / add tree
      std::vector<const u64 *> cts, pts; std::vector<int> sizes;
      for (auto &l : st.sum) {
        cts.push_back(A + p.vals[l.first->index].off);
        sizes.push_back(p.vals[l.first->index].size);
        pts.push_back(l.second ? A + p.vals[l.second->index].off : nullptr);
      }
      std::vector<int> kinds = st.sumKind;
      for (auto &lo : st.rotSums) { cts.push_back(A + p.rotSumOff(lo)); sizes.push_back(2); pts.push_back(nullptr); kinds.push_back(0); }
      check(evab_sum_products(c, o.ell, out, (int)cts.size(), cts.data(), sizes.data(), pts.data(), kinds.data(), stream));
      return;
    }
    auto V = [&](int i) -> const ValueInfo & { return p.vals[t.operandAt(i)->index]; };
    auto P = [&](int i) -> const u64 * { return A + p.vals[t.operandAt(i)->index].off; };
    switch (t.op) {
      case Op::Encode: {
        const EncodeGroup &g = p.groups[p.groupIndex.at(t.index)];
        if (g.first == &t && (g.dynamic || !p.opt.cacheConstants)) issueEncodeGroup(g, stream);
      } break;
      case Op::Add: case Op::Sub: case Op::Mul: {
        int ci = V(0).kind == Kind::Cipher ? 0 : 1, oi = 1 - ci;
        if (V(oi).kind == Kind::Cipher) {
          if (t.op == Op::Add) check(evab_add(c, o.ell, out, P(0), V(0).size, P(1), V(1).size, stream));
          else if (t.op == Op::Sub) check(evab_sub(c, o.ell, out, P(0), V(0).size, P(1), V(1).size, stream));
          else if (t.operandAt(0) == t.operandAt(1)) check(evab_square(c, o.ell, out, P(0), stream));  // seal_executor.h:161
          else check(evab_mul(c, o.ell, out, P(0), P(1), stream));
        } else {
          if (t.op == Op::Add) check(evab_add_plain(c, o.ell, out, P(ci), V(ci).size, P(oi), stream));
          else if (t.op == Op::Sub) check(evab_sub_plain(c, o.ell, out, P(0), V(0).size, P(1), stream));
          else check(evab_mul_plain(c, o.ell, out, P(ci), V(ci).size, P(oi), stream));
        }
      } break;
      case Op::Negate: check(evab_negate(c, o.ell, out, P(0), V(0).size, stream)); break;
      case Op::RotateLeftConst: case Op::RotateRightConst:
        if (*t.rotation == 0) check(evab_copy(c, o.ell, out, P(0), 2, stream));  // rotate_vector(0): copy
        else {
          const u64 elt = galoisElt(t);
          const u64 *in = A + p.vals[p.src(&t)->index].off;   // a composed rotation's last hop reads the hop before it
          if (st.hoist >= 0 && p.opt.hoistModUp)
            check(evab_rotate_modup_prepared(c, o.ell, out, in, A + p.hoistExtOff[st.hoist], elt, galoisKey(elt), hoistConst(elt, o.ell), work, stream));
          else if (st.hoist >= 0) check(evab_rotate_prepared(c, o.ell, out, in, A + p.hoistOff[st.hoist], elt, galoisKey(elt), work, stream));
          else check(evab_rotate(c, o.ell, out, in, elt, galoisKey(elt), work, stream));
        }
        break;
      case Op::Relinearize: check(evab_relinearize(c, o.ell, out, P(0), relinKey(), work, stream)); break;
      case Op::ModSwitch: check(evab_mod_switch(c, V(0).ell, out, P(0), V(0).size, stream)); break;
      case Op::Rescale: check(evab_rescale(c, V(0).ell, out, P(0), V(0).size, work, stream)); break;
      default: throw std::runtime_error(std::string("Unhandled op ") + opName(t.op));
    }
  }
  // fork from `stream` into the plan's streams, issue every step, join back
  void replay(void *stream) {
    const Plan &p = plan_;
    evab_ctx *c = dev_->ctx();
    BatchGuard bg(p.opt.batch, p.stride, p.rawStride);
    const std::int32_t *table = bank_ ? reinterpret_cast<const std::int32_t *>(keyTableDev_.get()) : nullptr;
    KeyBankGuard kg(table, bank_ ? bank_->stride() : 0);
    HoistInlineGuard hg(bank_ && bank_->inlineConstants());
    KeySeededGuard sg(bank_ && bank_->seededKeys());
    KeyC1Guard cg(c1Table() ? table + p.opt.batch : nullptr);
    void *forkEv = events_[p.numEvents + p.usedStreams];
    for (int b = 0; p.numFlags && b < p.opt.batch; b++)   // zero-coefficient flags of the shared mod-ups
      check(evab_memset_zero(c, arena_.get() + (std::size_t)b * p.stride + p.flagsOff, 8 * p.numFlags * 8, stream));
    check(evab_event_record(c, forkEv, stream));
    for (int s = 0; s < p.usedStreams; s++) check(evab_stream_wait_event(c, streams_[s], forkEv));
    for (auto &st : p.steps) {
      void *s = streams_[st.stream];
      for (int e : st.waits) check(evab_stream_wait_event(c, s, events_[e]));
      issue(st, s);
      if (st.record >= 0) check(evab_event_record(c, events_[st.record], s));
    }
    for (int s = 0; s < p.usedStreams; s++) {
      check(evab_event_record(c, events_[p.numEvents + s], streams_[s]));
      check(evab_stream_wait_event(c, stream, events_[p.numEvents + s]));
    }
  }
  void capture() {
    evab_ctx *c = dev_->ctx();
    if (graph_) { evab_graph_destroy(c, graph_); graph_ = nullptr; }
    if (!capStream_) { check(evab_stream_create(c, &capStream_)); streams_.push_back(capStream_); }
    check(evab_graph_begin(c, capStream_));
    try { replay(capStream_); } catch (...) { void *g = nullptr; evab_graph_end(c, capStream_, &g); throw; }
    check(evab_graph_end(c, capStream_, &graph_));
    graphValid_ = true;
  }

  std::shared_ptr<Device> dev_;
  const KeySet &keys_;
  const KeyBank *bank_;
  Program &prog_;
  Plan plan_;
  u64 N_;
  std::vector<std::vector<std::vector<double>>> rawsB_;   // [instance][term]
  std::map<std::pair<u64, int>, DBuf> hoistConst_;        // (galois element, ell) -> cadd [2][ell+1][N]
  u64 *hostFlags_ = nullptr;                              // page-locked copy of the flags of the last run
  DBuf keyTableDev_;                                      // bank-bound: int32 [batch] slots, then [batch] c1 entries (c1Table), read by the kernels
  std::int32_t *keyTableHost_ = nullptr;                  // its page-locked source (setKeyTable)
  std::unordered_set<std::uint64_t> rawUploaded_;
  bool staticEncoded_ = false;
  DBuf rawArena_;
  std::vector<void *> streams_, events_;
  void *capStream_ = nullptr;
  void *mainStream_ = nullptr;
  void *graph_ = nullptr;
  bool graphValid_ = false, rawDirty_ = false;
  DBuf arena_;
};

}  // namespace evab
