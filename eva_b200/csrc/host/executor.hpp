// executor.hpp -- GPU executor + stream/graph DAG scheduler for compiled EVA
// programs.  Replaces, for the hot path,
//   SEALExecutor::operator()/setInputs/getOutputs/free  (reference eva/seal/seal_executor.h:264-436)
//   ProgramTraversal / MulticoreProgramTraversal::forwardPass
//                                                       (eva/common/program_traversal.h:36-88,
//                                                        eva/common/multicore_program_traversal.h:24-84)
// Instead of interpreting the DAG term by term on CPU threads, the program is
// lowered ONCE into a static plan (value kinds, levels, scales, device buffer
// offsets, stream assignment, event edges); every execute() then replays the
// plan: independent terms run concurrently on different CUDA streams, cross-
// stream dependencies are events, and the whole replay can be captured into a
// CUDA graph so that one execute() costs a single graph launch.
#pragma once
#include "arena_packer.hpp"
#include "ckks_client.hpp"
#include "ir.hpp"
#include "logging.hpp"
#include <nvtx3/nvToolsExt.h>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <set>
#include <tuple>
#include <unordered_set>
#include <unordered_map>

namespace evab {

enum class Kind : int { None = 0, Cipher = 1, Plain = 2, Raw = 3 };

struct ValueInfo {
  Kind kind = Kind::None;
  int size = 0;        // ciphertext polynomials
  int ell = 0;         // residues
  double scale = 0.0;  // absolute scale (always an exact power of two in EVA)
  std::size_t off = 0; // word offset into the arena (Cipher / Plain)
  bool alias = false;  // shares its operand's storage (Output, step-0 rotation)
  bool fused = false;  // absorbed into a fused sum: the value is never materialised
};

struct Step {
  const Term *term;
  Op op;
  int stream = 0;
  std::vector<int> waits;  // event ids to wait for before issuing
  int record = -1;         // event id recorded after issuing
  std::size_t work = 0;    // scratch word offset in the stream's workspace (0 = none)
  // fused sum (root Add of a tree of cipher+cipher Adds): out = sum of ct (* pt when pt != null)
  std::vector<std::pair<const Term *, const Term *>> sum;
  std::vector<int> sumKind;    // per leaf: 0 ciphertext, 1 ciphertext * plaintext, 2 ciphertext (x) ciphertext
  int hoist = -1;              // rotation group sharing one inverse NTT (op == Undef: the step computing it)
  std::uint64_t producer = 0;  // term index, or termCount + group for a hoist step
  int lazy = -1;               // approxHoist / rotationSums: index of the rotation sums this pseudo step computes (op == Undef)
  int chunk = -1;              // rotationChunk: index of the rotation chunk this pseudo step computes (op == Undef)
  std::vector<std::size_t> lazyTemps;  // fused sum: arena offsets of the lazy rotation sums added to the other leaves
};

// Encode terms of one level that are encoded by a single batched device launch sequence
struct EncodeGroup {
  int ell; bool dynamic; std::vector<Term *> members; std::size_t outOff, workOff, rawOff; int stream = -1;
  Term *first = nullptr;   // earliest member in program order: its step issues the whole group
  int nUniform = 0;        // leading members whose vector is a replicated scalar: one-pass encoder
  bool withP = false;      // plaintexts of this group carry an extra residue row mod the key-switch prime (approxHoist)
};

// rotationChunk: up to 16 rotations of one hoist group computed by one evab_rotate_modup_many call (3 launches instead of 3 n)
struct RotChunk {
  int gid = 0, ell = 0;
  std::vector<const Term *> rots;
  std::size_t outOff = 0;                           // their results, contiguous: [n][2][ell][N]
  bool emitted = false;
};
// approxHoist: out_o = sum_i wts[o][i] (.) rots[i] over rotations of one hoist group, each sum rounded down by P once (evab_lazy_rotsum);
// rotationSums: the same sums with scalar-constant weights and every rotation rounded on its own, + sum_t twts[o][t] (.) taps[t] (evab_rotate_wsum)
struct LazySum {
  int gid = 0, ell = 0;
  std::vector<const Term *> rots;                   // union of the rotations (never materialised when all their uses are lazy)
  std::vector<const Term *> roots;                  // the fused sum every output feeds
  std::vector<std::vector<const Term *>> wts;       // [output][rotation]: plaintext weight, null when the rotation is not in that sum
  std::vector<const Term *> taps;                   // rotationSums: size-2 ciphertexts of the sums' other scalar-weighted leaves
  std::vector<std::vector<const Term *>> twts;      // [output][tap]: their weights, null when the tap is not in that sum
  std::size_t tempOff = 0;                          // arena offset of the outputs [nout][2][ell][N]
  bool emitted = false, allStatic = true;
};

struct ExecOptions {
  int numStreams = 8;
  bool useGraph = true;
  bool cacheConstants = true;  // encode plan-time-constant plaintexts once per plan instead of on every run
  int batch = 1;               // independent program instances executed by every (fat) kernel launch
  int fuse = 1;                // executeBatch: instances per plan replica (replicas run concurrently)
  std::map<std::string, int> inputSizes;   // ciphertext inputs that are not size 2 (partial sums of a sharded DAG)
  bool uniformEncode = true;   // replicated scalars are encoded by the one-pass encoder (evab_encode_uniform)
  bool hoistRotations = true;  // rotations of one ciphertext share the inverse NTT of its c1 (exact)
  bool hoistModUp = true;      // ... and the mod-up of its digits (exact, ops_impl.hpp hoisted_modup); a zero coefficient in a digit
                               // raises a flag and the caller redoes the run without this option (B200Public::executeMany)
  bool fuseSums = true;        // trees of Add over multiply_plain results / ciphertexts run as one kernel
  int rotationChunk = 16;      // with hoistModUp: rotations of one ciphertext computed per evab_rotate_modup_many call (same bits); < 2: one call each
  bool approxHoist = false;    // OPT-IN, NOT bit-exact (SURVEY 8f-4): sums of plaintext-weighted rotations of one ciphertext are rounded down by P
                               // once per sum instead of once per rotation (evab_lazy_rotsum); graded by the MSE criterion only
  bool rotationSums = true;    // with hoistModUp and fuseSums: leaves "rotation of a hoist group (x) scalar constant" of fused sums are summed by
                               // evab_rotate_wsum (same bits, 2 n + 2 nout ell transforms instead of n (2 + 2 ell)); approxHoist takes precedence
  bool dedupConstants = true;  // Encode terms of identical constants at the same (level, scale) share one plaintext
  bool dedupTerms = true;      // identical ciphertext terms (same op, same attributes, same operands) are evaluated once and
                               // aliased: the compiled wide DAG of tests/large_programs.py style repeats each of its 127
                               // distinct rotations 64 times.  Same bits; still counted as executed IR terms.
  std::size_t arenaLimit = 0;  // bytes a plan's arena may take (0: the free device memory at plan time).  A plan whose one-offset-per-
                               // value layout exceeds it reuses the storage of dead values (arena_packer.hpp); over it even then: error
};

// scoped evab_set_batch: ops issued by this thread act on `batch` instances
struct BatchGuard {
  BatchGuard(int batch, std::size_t stride, std::size_t vstride) { check(evab_set_batch(batch, stride, vstride)); }
  ~BatchGuard() { evab_set_batch(1, 0, 0); }
};

class Executor {
public:
  Executor(std::shared_ptr<Device> dev, CkksEncoder &enc, const KeySet &keys, Program &program, ExecOptions opt = {})
      : dev_(std::move(dev)), enc_(enc), keys_(keys), prog_(program), opt_(opt), N_(dev_->N()), k_(dev_->k()) {
    buildPlan();
  }
  ~Executor() {
    if (graph_) evab_graph_destroy(dev_->ctx(), graph_);
    if (hostFlags_) evab_host_free(hostFlags_);
    for (void *e : events_) evab_event_destroy(dev_->ctx(), e);
    for (void *s : streams_) evab_stream_destroy(dev_->ctx(), s);
  }
  Executor(const Executor &) = delete;

  std::size_t cipherOpCount() const { return cipherOps_; }
  // shape of the plan (test / tooling hook)
  std::map<std::string, long> planStats() const {
    std::map<std::string, long> m;
    m["steps"] = (long)steps_.size(); m["streams"] = usedStreams_; m["hoist_groups"] = (long)hoistOff_.size();
    m["rotation_chunks"] = (long)chunks_.size(); m["chunked_rotations"] = 0;
    const bool approx = opt_.approxHoist;   // lazy_ holds the approximate (lazy_*) or the exact (rotation_sum_*) calls
    m["lazy_calls"] = approx ? (long)lazy_.size() : 0; m["rotation_sum_calls"] = approx ? 0 : (long)lazy_.size();
    m["lazy_sums"] = m["lazy_rotations"] = m["rotation_sums"] = m["rotation_sum_rotations"] = m["rotation_sum_taps"] = 0;
    for (auto &L : lazy_) {
      m[approx ? "lazy_sums" : "rotation_sums"] += (long)L.roots.size();
      m[approx ? "lazy_rotations" : "rotation_sum_rotations"] += (long)L.rots.size();
      m["rotation_sum_taps"] += (long)L.taps.size();
    }
    for (auto &c : chunks_) m["chunked_rotations"] += (long)c.rots.size();
    long elided = 0;
    for (auto &t : order_) if ((t->op == Op::RotateLeftConst || t->op == Op::RotateRightConst) && vals_[t->index].fused) elided++;
    m["elided_rotations"] = elided;
    m["arena_bytes"] = (long)arenaBytes(); m["arena_bytes_unpacked"] = (long)unpackedBytes_; m["packed"] = packed_ ? 1 : 0;
    m["reuse_waits"] = reuseWaits_;
    long constWords = 0;   // plaintexts of plan-time constants, resident for the plan's lifetime
    if (opt_.cacheConstants)
      for (auto &g : groups_) if (!g.dynamic) constWords += (long)g.members.size() * (g.ell + (g.withP ? 1 : 0)) * (long)N_;
    m["constant_bytes"] = constWords * 8 * opt_.batch;
    return m;
  }
  // false when the plan's arena is packed and the value's storage may have been reused by a later value of the run
  bool intact(std::uint64_t index) const { return !packed_ || keptAfterRun_.at(index); }
  // private stream used by B200Public::execute for H2D -> run -> D2H of this plan,
  // so that execute() calls on different programs overlap on the GPU
  std::size_t arenaBytes() const { return (stride_ * (std::size_t)opt_.batch + 8 + rawStride_ * (std::size_t)opt_.batch + 8) * 8; }
  void *mainStream() {
    if (!mainStream_) { check(evab_stream_create(dev_->ctx(), &mainStream_)); streams_.push_back(mainStream_); }
    return mainStream_;
  }
  const ValueInfo &info(const Term::Ptr &t) const { return vals_.at(t->index); }
  int batch() const { return opt_.batch; }
  u64 *valuePtr(const Term::Ptr &t, int b = 0) const { return arena_.get() + (std::size_t)b * stride_ + vals_.at(t->index).off; }
  u64 *valuePtr(std::uint64_t index, int b = 0) const { return arena_.get() + (std::size_t)b * stride_ + vals_.at(index).off; }
  const ValueInfo &info(std::uint64_t index) const { return vals_.at(index); }
  const std::vector<double> &rawValue(std::uint64_t index, int b = 0) const { return rawsB_.at(b).at(index); }

  // device-resident run: inputs must already be in valuePtr(input term); raw
  // inputs set through setRawInput.  Enqueues the whole program on `stream`
  // (graph launch or multi-stream replay); does not synchronise.
  void run(void *stream) {
    if (rawDirty_) { evalRawAndEncodes(stream); rawDirty_ = false; }
    if (opt_.useGraph && verbosity() < 2) {   // debug verbosity: step-by-step replay so that every term is reported
      if (!graph_ || !graphValid_) capture();
      check(evab_graph_launch(dev_->ctx(), graph_, stream));
    } else {
      replay(stream);
    }
    for (int b = 0; numFlags_ && b < opt_.batch; b++)   // travels with the outputs; read by flagsRaised() once the stream is synchronised
      dev_->download(hostFlags_ + (std::size_t)b * 8 * numFlags_, arena_.get() + (std::size_t)b * stride_ + flagsOff_, 8 * numFlags_ * 8, stream);
  }
  // after the run's stream has been synchronised: did a digit of a rotation group hold a zero coefficient?  (The shared mod-up is
  // then not the reference's value; the caller must redo the run with hoistModUp off.  Probability ~ N ell 2^-60 per ciphertext.)
  bool flagsRaised() const {
    for (std::size_t i = 0; i < 8 * numFlags_ * (std::size_t)opt_.batch; i++)
      if (hostFlags_[i]) return true;
    return false;
  }
  void setRawInput(const std::string &name, const std::vector<double> &v, int b = 0) {
    auto t = prog_.getInput(name);
    if (vals_.at(t->index).kind != Kind::Raw) throw std::runtime_error("input " + name + " is not a raw input");
    std::vector<double> x;
    ConstantValue(prog_.getVecSize(), v).expandTo(x, prog_.getVecSize());
    rawsB_.at(b)[t->index] = x;
    rawDirty_ = true;
  }

private:
  // ---------------------------------------------------------------- planning
  void buildPlan() {
    for (auto &t : prog_.toposort()) order_.push_back(t.get());  // raw: the plan lives inside the Program (attachment)
    vals_.assign(prog_.termCount(), ValueInfo{});
    if (opt_.batch < 1) throw std::invalid_argument("batch must be >= 1");
    rawsB_.assign(opt_.batch, std::vector<std::vector<double>>(prog_.termCount()));
    std::size_t arenaWords = 0;
    auto place = [&](ValueInfo &v) { v.off = arenaWords; arenaWords += (std::size_t)(v.kind == Kind::Cipher ? v.size : 1) * v.ell * N_; };
    byIndex_.assign(prog_.termCount(), nullptr);
    canon_.resize(prog_.termCount());
    for (std::size_t i = 0; i < canon_.size(); i++) canon_[i] = i;
    std::map<std::tuple<int, long long, std::uint64_t, std::uint64_t>, std::uint64_t> seenTerm;
    for (auto &t : order_) {
      ValueInfo &v = vals_[t->index];
      byIndex_[t->index] = t;
      auto a = [&](int i) -> const ValueInfo & { return vals_[t->operandAt(i)->index]; };
      if (opt_.dedupTerms && t->numOperands() >= 1 && vals_[t->operandAt(0)->index].kind != Kind::Raw &&
          (t->op == Op::Add || t->op == Op::Sub || t->op == Op::Mul || t->op == Op::Negate || t->op == Op::RotateLeftConst ||
           t->op == Op::RotateRightConst || t->op == Op::Relinearize || t->op == Op::ModSwitch || t->op == Op::Rescale)) {
        const long long attr = t->rotation ? (long long)*t->rotation : (t->rescaleDivisor ? (long long)*t->rescaleDivisor : 0);
        const std::uint64_t o0 = canon_[t->operandAt(0)->index], o1 = t->numOperands() > 1 ? canon_[t->operandAt(1)->index] : ~0ull;
        auto ins = seenTerm.emplace(std::make_tuple((int)t->op, attr, o0, o1), t->index);
        if (!ins.second && vals_[ins.first->second].kind == Kind::Cipher) {
          canon_[t->index] = ins.first->second;
          v = vals_[ins.first->second]; v.alias = true;     // same value: shares the first occurrence's storage
          cipherOps_++;                                      // still an executed IR term of the program
          continue;
        }
      }
      switch (t->op) {
        case Op::Input: {
          const Type ty = t->type.value_or(Type::Cipher);
          if (ty == Type::Raw) { v.kind = Kind::Raw; rawInputs_ = true; break; }
          if (!t->encodeAtScale || !t->encodeAtLevel) throw std::runtime_error("input term lacks scale/level (program not compiled?)");
          v.kind = ty == Type::Cipher ? Kind::Cipher : Kind::Plain;
          v.size = 2; v.ell = levelToEll(*t->encodeAtLevel); v.scale = std::ldexp(1.0, (int)*t->encodeAtScale);
          if (v.kind == Kind::Cipher && !opt_.inputSizes.empty())
            for (auto &in : prog_.getInputs())
              if (in.second.get() == t) { auto f = opt_.inputSizes.find(in.first); if (f != opt_.inputSizes.end()) v.size = f->second; }
          if (v.size < 2 || v.size > 3) throw std::runtime_error("input ciphertext size must be 2 or 3");
          place(v);
        } break;
        case Op::Constant:
          v.kind = Kind::Raw;
          for (auto &r : rawsB_) t->constant->expandTo(r[t->index], prog_.getVecSize());
          break;
        case Op::Encode:
          if (a(0).kind != Kind::Raw) throw std::runtime_error("Encode expects a raw operand");
          v.kind = Kind::Plain; v.ell = levelToEll(t->encodeAtLevel.value()); v.scale = std::ldexp(1.0, (int)t->encodeAtScale.value());
          encodeTerms_.push_back(t);   // placed below, contiguous per (level, static/dynamic) group
          break;
        case Op::Add: case Op::Sub: case Op::Mul: {
          const ValueInfo &x = a(0), &y = a(1);
          if (x.kind == Kind::Raw && y.kind == Kind::Raw) { v.kind = Kind::Raw; break; }
          if (x.kind == Kind::Raw || y.kind == Kind::Raw) throw std::runtime_error("Unsupported operation encountered");
          if (x.kind != Kind::Cipher && y.kind != Kind::Cipher) throw std::runtime_error("Unsupported operation encountered");
          if (x.ell != y.ell) throw std::invalid_argument("encrypted1 and encrypted2 parameter mismatch");
          const ValueInfo &c = x.kind == Kind::Cipher ? x : y, &o = x.kind == Kind::Cipher ? y : x;
          v.kind = Kind::Cipher; v.ell = x.ell;
          if (t->op == Op::Mul) {
            v.scale = x.scale * y.scale;
            if (o.kind == Kind::Cipher) {
              if (x.size != 2 || y.size != 2) throw std::runtime_error("ciphertext multiplication expects size-2 operands");
              v.size = 3;
            } else v.size = c.size;
          } else {
            if (x.scale != y.scale) throw std::invalid_argument("scale mismatch");
            v.scale = x.scale;
            v.size = o.kind == Kind::Cipher ? std::max(x.size, y.size) : c.size;
            if (t->op == Op::Sub && x.kind != Kind::Cipher) throw std::runtime_error("plain - cipher must be lowered before execution");
          }
          place(v);
        } break;
        case Op::Negate:
          if (a(0).kind == Kind::Raw) { v.kind = Kind::Raw; break; }
          v = a(0); v.alias = false; place(v);
          break;
        case Op::RotateLeftConst: case Op::RotateRightConst:
          if (a(0).kind == Kind::Raw) { v.kind = Kind::Raw; break; }
          if (a(0).kind != Kind::Cipher || a(0).size != 2) throw std::runtime_error("rotation expects a size-2 ciphertext");
          v = a(0); v.alias = false; place(v);
          break;
        case Op::Relinearize:
          if (a(0).kind != Kind::Cipher) throw std::runtime_error("Relinearize expects a ciphertext");
          v = a(0); v.alias = false; v.size = 2; place(v);
          break;
        case Op::ModSwitch: case Op::Rescale:
          if (a(0).kind != Kind::Cipher) throw std::runtime_error("ModSwitch/Rescale expects a ciphertext");
          if (a(0).ell < 2) throw std::invalid_argument("end of modulus switching chain reached");
          v = a(0); v.alias = false; v.ell = a(0).ell - 1;
          if (t->op == Op::Rescale) v.scale = a(0).scale / std::ldexp(1.0, (int)t->rescaleDivisor.value());
          place(v);
          break;
        case Op::Output:
          v = a(0); v.alias = true;
          break;
        default: throw std::runtime_error(std::string("Unhandled op ") + opName(t->op));
      }
      if (v.kind == Kind::Cipher && t->op != Op::Input && t->op != Op::Output) cipherOps_++;
    }
    // ---- fused sums: a tree of cipher+cipher Adds whose inner nodes have a single use collapses into
    // one kernel; leaves that are single-use multiply_plain results are multiplied on the fly
    // (Sobel / Harris filter taps: sum_i rot_i(x) * w_i).  Same canonical result, see evab_sum_terms.
    std::unordered_map<std::uint64_t, std::vector<std::pair<const Term *, const Term *>>> sumOf;
    std::unordered_map<std::uint64_t, std::vector<int>> sumKindOf;
    if (opt_.fuseSums) {
      std::vector<int> uses(prog_.termCount(), 0);
      for (auto &t : order_) if (canon_[t->index] == t->index) for (auto &o : t->getOperands()) uses[canon_[o->index]]++;
      auto isCipherAdd = [&](const Term *t) {
        return t->op == Op::Add && vals_[t->operandAt(0)->index].kind == Kind::Cipher && vals_[t->operandAt(1)->index].kind == Kind::Cipher;
      };
      auto plainMul = [&](const Term *t, const Term *&ct, const Term *&pt) {
        if (t->op != Op::Mul) return false;
        const Term *a = C(t->operandAt(0).get()), *b = C(t->operandAt(1).get());
        if (vals_[a->index].kind == Kind::Cipher && vals_[b->index].kind == Kind::Plain) { ct = a; pt = b; return true; }
        if (vals_[b->index].kind == Kind::Cipher && vals_[a->index].kind == Kind::Plain) { ct = b; pt = a; return true; }
        return false;
      };
      // Evaluator::multiply / square of two size-2 ciphertexts (2x2 -> 3)
      auto cipherMul = [&](const Term *t, const Term *&a, const Term *&b) {
        if (t->op != Op::Mul) return false;
        a = C(t->operandAt(0).get()); b = C(t->operandAt(1).get());
        return vals_[a->index].kind == Kind::Cipher && vals_[b->index].kind == Kind::Cipher && vals_[a->index].size == 2 && vals_[b->index].size == 2;
      };
      for (auto it = order_.rbegin(); it != order_.rend(); ++it) {
        Term *root = *it;
        if (!isCipherAdd(root) || vals_[root->index].fused || vals_[root->index].alias) continue;
        std::vector<std::pair<const Term *, const Term *>> leaves;
        std::vector<int> kinds;
        std::vector<const Term *> absorbed;
        std::function<void(const Term *)> expand = [&](const Term *t) {
          const Term *ct = nullptr, *pt = nullptr;
          const bool inner = t != root;
          if ((!inner || uses[t->index] == 1) && isCipherAdd(t) && leaves.size() + 2 <= 30) {
            if (inner) absorbed.push_back(t);
            expand(C(t->operandAt(0).get()));
            expand(C(t->operandAt(1).get()));
          } else if (inner && uses[t->index] == 1 && plainMul(t, ct, pt)) {
            absorbed.push_back(t);
            leaves.emplace_back(ct, pt); kinds.push_back(1);
          } else if (inner && uses[t->index] == 1 && cipherMul(t, ct, pt)) {
            absorbed.push_back(t);
            leaves.emplace_back(ct, pt); kinds.push_back(2);
          } else {
            leaves.emplace_back(t, nullptr); kinds.push_back(0);
          }
        };
        expand(root);
        if (absorbed.empty() || leaves.size() > 32) continue;   // a plain two-operand add
        for (const Term *t : absorbed) vals_[t->index].fused = true;
        sumOf[root->index] = std::move(leaves);
        sumKindOf[root->index] = std::move(kinds);
      }
    }
    // operands a step really reads (fused sums read their leaves)
    auto stepOperands = [&](const Term *t) {
      std::vector<const Term *> ops;
      auto f = sumOf.find(t->index);
      if (f == sumOf.end()) { for (auto &o : t->getOperands()) ops.push_back(C(o.get())); return ops; }
      for (auto &l : f->second) { ops.push_back(l.first); if (l.second) ops.push_back(l.second); }
      return ops;
    };
    // ---- hoisted rotations: two or more rotations of the same ciphertext share the inverse NTT of
    // its c1 (evab_rotate_prepare); the shared buffer is produced by a pseudo step of its own
    const std::uint64_t TC = prog_.termCount();
    std::unordered_map<std::uint64_t, int> hoistOf;       // rotation term -> group
    std::vector<const Term *> hoistSrc;
    if (opt_.hoistRotations) {
      std::map<std::uint64_t, std::vector<const Term *>> bySrc;
      for (auto &t : order_)
        if ((t->op == Op::RotateLeftConst || t->op == Op::RotateRightConst) && *t->rotation != 0 && vals_[t->index].kind == Kind::Cipher &&
            vals_[t->index].ell <= 15 && !vals_[t->index].alias)
          bySrc[canon_[t->operandAt(0)->index]].push_back(t);
      for (auto &kv : bySrc) {
        if (kv.second.size() < 2) continue;
        const int gid = (int)hoistSrc.size();
        hoistSrc.push_back(C(kv.second.front()->operandAt(0).get()));
        hoistOff_.push_back(arenaWords);
        arenaWords += (std::size_t)vals_[kv.first].ell * N_;
        if (opt_.hoistModUp) {   // the extended digits [ell+1][ell][N], shared by the rotations of this ciphertext
          hoistExtOff_.push_back(arenaWords);
          arenaWords += evab_rotate_modup_ext_bytes(dev_->ctx(), vals_[kv.first].ell) / 8;
        }
        for (const Term *r : kv.second) hoistOf[r->index] = gid;
      }
    }
    // ---- rotation sums.  approxHoist (opt-in): leaves "rotation of a hoist group (x) constant plaintext" of a fused sum, two or more
    // of the same group, become ONE lazy rotation sum whose temporary joins the remaining leaves; a rotation all of whose uses went that
    // way is never materialised.  The plaintexts involved are encoded with an extra residue row mod P.
    // rotationSums (exact, evab_rotate_wsum): the same grouping, for rotations whose every use is such a leaf with a scalar constant
    // weight.  A leaf of weight 0.0 is dropped (its product is the zero ciphertext), and the sum's other leaves "size-2 ciphertext
    // (x) scalar constant" join the call as taps (a rotation by 0 through its operand).  A sum left with no other leaf is the call's
    // output itself: it is never issued as a step of its own.
    const bool exactSums = !opt_.approxHoist && opt_.rotationSums;
    if ((opt_.approxHoist || exactSums) && opt_.hoistModUp && opt_.fuseSums) {
      std::vector<int> usesAll(prog_.termCount(), 0), lazyUses(prog_.termCount(), 0), wsumLeaves(prog_.termCount(), 0), pos(prog_.termCount(), 0);
      for (auto &t : order_) if (canon_[t->index] == t->index) for (auto &o : t->getOperands()) usesAll[canon_[o->index]]++;
      for (std::size_t i = 0; i < order_.size(); i++) pos[order_[i]->index] = (int)i;
      // a replicated scalar constant (the uniform encoder's predicate) and its value
      auto scalarWeight = [&](const Term *pt, double &v) {
        if (pt->op != Op::Encode || pt->operandAt(0)->op != Op::Constant) return false;
        const auto &x = rawsB_[0][pt->operandAt(0)->index];
        if (x.empty() || !std::all_of(x.begin(), x.end(), [&](double y) { return std::memcmp(&y, &x[0], sizeof(double)) == 0; })) return false;
        v = x[0];
        return true;
      };
      auto rotLeaf = [&](const std::pair<const Term *, const Term *> &l) {
        double v;
        return hoistOf.count(l.first->index) && vals_[l.first->index].size == 2 && (exactSums ? scalarWeight(l.second, v) : l.second->op == Op::Encode);
      };
      if (exactSums)
        for (auto &kv : sumOf)
          for (std::size_t i = 0; i < kv.second.size(); i++)
            if (sumKindOf.at(kv.first)[i] == 1 && rotLeaf(kv.second[i])) wsumLeaves[kv.second[i].first->index]++;
      std::map<int, int> openOf;   // hoist group -> the lazy sum that still takes outputs
      for (auto &t : order_) {
        auto f = sumOf.find(t->index);
        if (f == sumOf.end()) continue;
        auto &leaves = f->second;
        auto &kinds = sumKindOf.at(t->index);
        std::map<int, std::vector<int>> byGroup;
        for (int i = 0; i < (int)leaves.size(); i++) {
          if (kinds[i] != 1 || !rotLeaf(leaves[i])) continue;
          if (exactSums && wsumLeaves[leaves[i].first->index] != usesAll[leaves[i].first->index]) continue;
          byGroup[hoistOf.at(leaves[i].first->index)].push_back(i);
        }
        auto isZero = [&](int i) { double v = 1.0; return exactSums && scalarWeight(leaves[i].second, v) && v == 0.0; };
        std::vector<char> drop(leaves.size(), 0);
        std::vector<std::pair<int, std::vector<int>>> slices;   // at most 16 rotations per call: longer sums are cut
        for (auto &kv : byGroup)
          for (std::size_t b = 0; b < kv.second.size(); b += 16)
            slices.emplace_back(kv.first, std::vector<int>(kv.second.begin() + b, kv.second.begin() + std::min(kv.second.size(), b + 16)));
        for (auto &kv : slices) {
          if (kv.second.size() < 2 || std::all_of(kv.second.begin(), kv.second.end(), isZero)) continue;
          // sums over rotations of the same ciphertext share one call (and the inner products of the rotations they have in
          // common), as long as the later sum's weights are available when the first one runs
          int li = -1;
          if (auto op = openOf.find(kv.first); op != openOf.end()) {
            LazySum &L = lazy_[op->second];
            // (constants of one level are encoded together, before the first of them is used: every weight is ready by then)
            std::size_t extra = 0;
            bool ready = L.roots.size() < 4 && L.allStatic;
            for (int i : kv.second) {
              if (!isZero(i) && std::find(L.rots.begin(), L.rots.end(), leaves[i].first) == L.rots.end()) extra++;
              if (leaves[i].second->operandAt(0)->op != Op::Constant) ready = false;
            }
            if (ready && L.rots.size() + extra <= 16) li = op->second;
          }
          if (li < 0) {
            li = (int)lazy_.size();
            lazy_.emplace_back();
            lazy_[li].gid = kv.first; lazy_[li].ell = vals_[t->index].ell;
            openOf[kv.first] = li;
          }
          LazySum &L = lazy_[li];
          L.roots.push_back(t);
          for (auto &w : L.wts) w.resize(L.rots.size(), nullptr);
          L.wts.emplace_back(L.rots.size(), nullptr);
          L.twts.emplace_back(L.taps.size(), nullptr);
          for (int i : kv.second) {
            if (isZero(i)) { drop[i] = 1; lazyUses[leaves[i].first->index]++; continue; }
            auto r = std::find(L.rots.begin(), L.rots.end(), leaves[i].first);
            if (r == L.rots.end()) { L.rots.push_back(leaves[i].first); for (auto &w : L.wts) w.push_back(nullptr); r = L.rots.end() - 1; }
            auto &slot = L.wts.back()[r - L.rots.begin()];
            if (slot) continue;   // the same rotation twice in one sum: the second one stays an ordinary leaf
            slot = leaves[i].second;
            if (slot->operandAt(0)->op != Op::Constant) L.allStatic = false;
            drop[i] = 1; lazyUses[leaves[i].first->index]++;
            if (!exactSums) needP_.insert(leaves[i].second->index);
          }
          lazyOfRoot_[t->index].emplace_back(li, (int)L.roots.size() - 1);
        }
        if (!lazyOfRoot_.count(t->index)) continue;
        if (exactSums) {   // the other scalar-weighted leaves: taps of the first call, when they are computed before that call is issued
          const auto [li, o] = lazyOfRoot_.at(t->index).front();
          LazySum &L = lazy_[li];
          for (int i = 0; i < (int)leaves.size(); i++) {
            double v;
            if (drop[i] || kinds[i] != 1 || vals_[leaves[i].first->index].size != 2 || !scalarWeight(leaves[i].second, v)) continue;
            const Term *ct = leaves[i].first;
            const bool rot0 = (ct->op == Op::RotateLeftConst || ct->op == Op::RotateRightConst) && *ct->rotation == 0;
            const Term *src = rot0 ? C(ct->operandAt(0).get()) : ct;
            if (vals_[src->index].fused || pos[src->index] >= pos[L.roots.front()->index]) continue;
            if (v == 0.0) { drop[i] = 1; if (rot0) lazyUses[ct->index]++; continue; }
            auto tp = std::find(L.taps.begin(), L.taps.end(), src);
            if (tp == L.taps.end()) {
              if (L.taps.size() >= 16) continue;
              L.taps.push_back(src); for (auto &w : L.twts) w.push_back(nullptr); tp = L.taps.end() - 1;
            }
            auto &slot = L.twts[o][tp - L.taps.begin()];
            if (slot) continue;
            slot = leaves[i].second;
            drop[i] = 1;
            if (rot0) lazyUses[ct->index]++;   // read through its operand: the copy itself may never be made
          }
        }
        std::vector<std::pair<const Term *, const Term *>> keep; std::vector<int> keepKind;
        for (int i = 0; i < (int)leaves.size(); i++) if (!drop[i]) { keep.push_back(leaves[i]); keepKind.push_back(kinds[i]); }
        leaves = std::move(keep); kinds = std::move(keepKind);
        if (exactSums && leaves.empty() && lazyOfRoot_.at(t->index).size() == 1) directOf_[t->index] = lazyOfRoot_.at(t->index).front();
      }
      for (auto &L : lazy_) { L.tempOff = arenaWords; arenaWords += L.roots.size() * 2 * (std::size_t)L.ell * N_; }
      for (auto &kv : directOf_) vals_[kv.first].off = lazy_[kv.second.first].tempOff + (std::size_t)kv.second.second * 2 * lazy_[kv.second.first].ell * N_;
      for (auto &t : order_)
        if (lazyUses[t->index] && lazyUses[t->index] == usesAll[t->index]) vals_[t->index].fused = true;   // the rotation is never materialised
    }
    // ---- batched rotations: the (materialised) rotations of a hoist group are computed together, 16 per call
    if (opt_.rotationChunk >= 2 && opt_.hoistModUp) {
      std::vector<int> open(hoistSrc.size(), -1);
      for (auto &t : order_) {
        auto h = hoistOf.find(t->index);
        if (h == hoistOf.end() || vals_[t->index].fused || canon_[t->index] != t->index) continue;
        int ci = open[h->second];
        if (ci < 0 || (int)chunks_[ci].rots.size() >= std::min(16, opt_.rotationChunk)) {
          ci = open[h->second] = (int)chunks_.size();
          chunks_.emplace_back();
          chunks_[ci].gid = h->second; chunks_[ci].ell = vals_[t->index].ell;
        }
        chunkOf_[t->index] = ci;
        chunks_[ci].rots.push_back(t);
      }
      for (auto &ch : chunks_) {
        ch.outOff = arenaWords;
        for (std::size_t i = 0; i < ch.rots.size(); i++) vals_[ch.rots[i]->index].off = arenaWords + i * 2 * (std::size_t)ch.ell * N_;
        arenaWords += ch.rots.size() * 2 * (std::size_t)ch.ell * N_;
      }
    }
    // ---- Encode groups: one batched device encode per (ell, input-dependent?) group.
    // Static groups (constants only) are encoded once per plan when cacheConstants is
    // set, otherwise every run like the reference (seal_executor.h:303-308).
    {
      std::vector<char> dyn(prog_.termCount(), 0);
      for (auto &t : order_) {
        bool d = (t->op == Op::Input && vals_[t->index].kind == Kind::Raw);
        for (auto &o : t->getOperands()) d = d || dyn[o->index];
        dyn[t->index] = d;
      }
      std::map<std::tuple<int, int, int>, int> groupOf;
      // identical constant vectors encoded at the same level and scale give identical plaintexts:
      // later occurrences alias the first one (same bits as encoding each, seal_executor.h:217-248)
      std::map<std::tuple<int, double, std::vector<double>, int>, Term *> firstOf;
      for (Term *t : encodeTerms_) {
        if (opt_.dedupConstants && !dyn[t->index] && t->operandAt(0)->op == Op::Constant) {
          auto ck = std::make_tuple(vals_[t->index].ell, vals_[t->index].scale, rawsB_[0][t->operandAt(0)->index], (int)needP_.count(t->index));
          auto ins = firstOf.emplace(std::move(ck), t);
          if (!ins.second) {
            encodeAlias_[t->index] = ins.first->second;
            groupIndex_[t->index] = groupIndex_.at(ins.first->second->index);
            continue;
          }
        }
        auto key = std::make_tuple(vals_[t->index].ell, (int)dyn[t->index], (int)needP_.count(t->index));
        auto it = groupOf.find(key);
        if (it == groupOf.end()) {
          it = groupOf.emplace(key, (int)groups_.size()).first;
          groups_.push_back(EncodeGroup{std::get<0>(key), std::get<1>(key) != 0, {}, 0, 0, 0});
          groups_.back().withP = std::get<2>(key) != 0;
        }
        groups_[it->second].members.push_back(t);
        groupIndex_[t->index] = it->second;
      }
      for (auto &g : groups_) {
        g.first = g.members.front();
        if (!g.dynamic && opt_.uniformEncode) {   // scalar constants first: they go through evab_encode_uniform
          auto uniform = [&](Term *t) {
            const auto &x = rawsB_[0][t->operandAt(0)->index];
            return !x.empty() && std::all_of(x.begin(), x.end(), [&](double v) { return std::memcmp(&v, &x[0], sizeof(double)) == 0; });
          };
          auto mid = std::stable_partition(g.members.begin(), g.members.end(), uniform);
          g.nUniform = (int)(mid - g.members.begin());
        }
        g.outOff = arenaWords;
        for (Term *t : g.members) { vals_[t->index].off = arenaWords; arenaWords += (std::size_t)(g.ell + (g.withP ? 1 : 0)) * N_; }
        g.workOff = arenaWords; arenaWords += evab_encode_work_bytes(dev_->ctx(), (int)g.members.size() - g.nUniform) / 8;
        g.rawOff = rawWords_;
        for (Term *t : g.members) { rawOff_[t->index] = rawWords_; rawWords_ += prog_.getVecSize(); }
      }
      for (auto &kv : encodeAlias_) vals_[kv.first].off = vals_[kv.second->index].off;
    }
    if (opt_.hoistModUp && !hoistSrc.empty()) {   // one zero-coefficient flag per group (64 bytes apart: no false sharing of the atomics)
      flagsOff_ = arenaWords; numFlags_ = hoistSrc.size();
      arenaWords += 8 * numFlags_;
    }
    // ---- stream assignment + event edges.  Producers are identified by term index, or TC + group
    // for the hoist pseudo steps.
    const int S = std::max(1, opt_.numStreams);
    const std::size_t NP = TC + hoistSrc.size() + lazy_.size() + chunks_.size();
    std::unordered_map<std::uint64_t, std::uint64_t> prodOf;   // rotation term -> the chunk step that produces it
    std::vector<int> streamOf(NP, -1), eventOf(NP, -1);
    std::vector<char> chainTaken(NP, 0), hoistDone(hoistSrc.size(), 0);
    std::vector<std::size_t> workWords(S, 0);
    int rr = 0;
    std::vector<char> inputTerm(NP, 0);
    for (auto &t : order_) if (t->op == Op::Input) inputTerm[t->index] = 1;
    auto isInput = [&](std::uint64_t id) { return inputTerm[id] != 0; };
    // place one step: continue the chain of a device operand nobody continued yet, else take a new
    // stream round-robin; cross-stream operands become event waits
    auto emit = [&](Step st, std::vector<std::uint64_t> operands, int forced, std::size_t w) {
      for (auto &o : operands) if (auto p = prodOf.find(o); p != prodOf.end()) o = p->second;
      int chosen = forced;
      for (std::uint64_t o : operands) {
        const int so = streamOf[o];
        if (so >= 0 && !chainTaken[o] && !isInput(o)) { chosen = so; chainTaken[o] = 1; break; }
      }
      if (chosen < 0) chosen = (rr++) % S;
      st.stream = chosen;
      for (std::uint64_t o : operands) {
        const int so = streamOf[o];
        if (so >= 0 && so != chosen && !isInput(o)) {
          if (eventOf[o] < 0) { eventOf[o] = numEvents_++; recordAfter_[o] = eventOf[o]; }
          if (std::find(st.waits.begin(), st.waits.end(), eventOf[o]) == st.waits.end()) st.waits.push_back(eventOf[o]);
        }
      }
      workWords[chosen] = std::max(workWords[chosen], w);
      streamOf[st.producer] = chosen;
      steps_.push_back(st);
    };
    // the pseudo step of a rotation sum call, issued before the first fused sum it feeds
    auto emitLazy = [&](int li) {
      LazySum &Lz = lazy_[li];
      const std::uint64_t lid = TC + hoistSrc.size() + (std::size_t)li;
      if (Lz.emitted) return lid;
      if (!hoistDone[Lz.gid]) {
        Step hs;
        hs.term = hoistSrc[Lz.gid]; hs.op = Op::Undef; hs.hoist = Lz.gid; hs.producer = TC + Lz.gid;
        emit(hs, {hoistSrc[Lz.gid]->index}, -1, 0);
        hoistDone[Lz.gid] = 1;
      }
      Step ls;
      ls.term = hoistSrc[Lz.gid]; ls.op = Op::Undef; ls.lazy = li; ls.producer = lid;
      std::vector<std::uint64_t> lops{hoistSrc[Lz.gid]->index, TC + (std::uint64_t)Lz.gid};
      for (auto &ws : Lz.wts) for (const Term *w : ws) if (w && streamOf[w->index] >= 0) lops.push_back(w->index);   // (later sums' constants: same encode group)
      for (auto &ws : Lz.twts) for (const Term *w : ws) if (w && streamOf[w->index] >= 0) lops.push_back(w->index);
      for (const Term *x : Lz.taps) lops.push_back(x->index);
      const std::size_t work = exactSums ? evab_rotate_wsum_work_bytes(dev_->ctx(), Lz.ell, (int)Lz.rots.size(), (int)Lz.roots.size())
                                         : evab_lazy_rotsum_work_bytes(dev_->ctx(), Lz.ell, (int)Lz.roots.size());
      emit(ls, lops, -1, work / 8);
      Lz.emitted = true;
      return lid;
    };
    for (auto &t : order_) {
      const ValueInfo &v = vals_[t->index];
      const bool device = (v.kind == Kind::Cipher || v.kind == Kind::Plain) && t->op != Op::Input && !v.alias && !v.fused;
      if (!device) {
        if (v.alias) streamOf[t->index] = streamOf[aliasSource(t)];
        continue;
      }
      if (auto d = directOf_.find(t->index); d != directOf_.end()) {   // the sum is a rotation sum call's output
        const std::uint64_t lid = emitLazy(d->second.first);
        prodOf[t->index] = lid; streamOf[t->index] = streamOf[lid];
        continue;
      }
      Step st;
      st.term = t; st.op = t->op; st.producer = t->index;
      { auto f = sumOf.find(t->index); if (f != sumOf.end()) { st.sum = f->second; st.sumKind = sumKindOf.at(t->index); } }
      std::vector<std::uint64_t> operands;
      for (const Term *o : stepOperands(t)) operands.push_back(o->index);
      if (auto lz = lazyOfRoot_.find(t->index); lz != lazyOfRoot_.end())
        for (auto &lo : lz->second) {   // the lazy rotation sums feeding this fused sum go first, as a pseudo step of their own
          const std::uint64_t lid = emitLazy(lo.first);
          st.lazyTemps.push_back(lazy_[lo.first].tempOff + (std::size_t)lo.second * 2 * lazy_[lo.first].ell * N_);
          operands.push_back(lid);
        }
      int forced = -1;
      if (t->op == Op::Encode) {
        EncodeGroup &g = groups_[groupIndex_.at(t->index)];
        if (g.stream < 0) g.stream = (rr++) % S;
        forced = g.stream;
      }
      std::size_t w = 0;
      if (t->op == Op::Relinearize || ((t->op == Op::RotateLeftConst || t->op == Op::RotateRightConst) && *t->rotation != 0))
        w = evab_keyswitch_work_bytes(dev_->ctx(), vals_[t->operandAt(0)->index].ell) / 8;
      else if (t->op == Op::Rescale)
        w = evab_rescale_work_bytes(dev_->ctx(), vals_[t->operandAt(0)->index].size) / 8;
      if (auto co = chunkOf_.find(t->index); co != chunkOf_.end()) {   // computed with the other rotations of its chunk
        RotChunk &ch = chunks_[co->second];
        const std::uint64_t cid = TC + hoistSrc.size() + lazy_.size() + (std::size_t)co->second;
        if (!ch.emitted) {
          if (!hoistDone[ch.gid]) {
            Step hs;
            hs.term = hoistSrc[ch.gid]; hs.op = Op::Undef; hs.hoist = ch.gid; hs.producer = TC + ch.gid;
            emit(hs, {hoistSrc[ch.gid]->index}, -1, 0);
            hoistDone[ch.gid] = 1;
          }
          Step cs;
          cs.term = hoistSrc[ch.gid]; cs.op = Op::Undef; cs.chunk = co->second; cs.hoist = ch.gid; cs.producer = cid;
          emit(cs, {hoistSrc[ch.gid]->index, TC + (std::uint64_t)ch.gid}, -1, evab_rotate_modup_many_work_bytes(dev_->ctx(), ch.ell, (int)ch.rots.size()) / 8);
          ch.emitted = true;
          for (const Term *r : ch.rots) { prodOf[r->index] = cid; streamOf[r->index] = streamOf[cid]; }
        }
        continue;
      }
      auto h = hoistOf.find(t->index);
      if (h != hoistOf.end()) {
        const int gid = h->second;
        if (!hoistDone[gid]) {   // first rotation of the group in program order: the shared inverse NTT goes first
          Step hs;
          hs.term = hoistSrc[gid]; hs.op = Op::Undef; hs.hoist = gid; hs.producer = TC + gid;
          emit(hs, {hoistSrc[gid]->index}, -1, 0);
          hoistDone[gid] = 1;
        }
        st.hoist = gid;
        operands.push_back(TC + gid);
      }
      emit(st, operands, forced, w);
    }
    // resolve alias chains (Output of X shares X's storage; Output(Output) never occurs)
    for (auto &t : order_) {
      ValueInfo &v = vals_[t->index];
      if (v.alias) { const ValueInfo &src = vals_[aliasSource(t)]; v.off = src.off; }
    }
    for (auto &st : steps_) {
      auto it = recordAfter_.find(st.producer);
      if (it != recordAfter_.end()) st.record = it->second;
    }
    // last step of every stream must be joined back into the caller's stream
    usedStreams_ = 0;
    for (auto &st : steps_) usedStreams_ = std::max(usedStreams_, st.stream + 1);
    workOff_.assign(usedStreams_, 0);
    for (int s = 0; s < usedStreams_; s++) { workOff_[s] = arenaWords; arenaWords += workWords[s]; }
    stride_ = (arenaWords + 63) & ~std::size_t(63);
    rawStride_ = (rawWords_ + 7) & ~std::size_t(7);
    // ---- arena layout: one offset per value (above) when it fits the limit, else the storage of dead values is reused
    unpackedBytes_ = arenaBytes();
    std::size_t limit = opt_.arenaLimit;
    if (!limit) { std::size_t freeB = 0, totalB = 0; check(evab_mem_info(dev_->ctx(), &freeB, &totalB)); limit = freeB; }
    if (unpackedBytes_ > limit) {
      packLayout(hoistSrc, workWords, stepOperands);
      if (arenaBytes() > limit)
        throw std::runtime_error("plan arena needs " + std::to_string(arenaBytes()) + " bytes packed (" + std::to_string(unpackedBytes_) +
                                 " bytes unpacked), more than the limit of " + std::to_string(limit) + " bytes");
    }
    arena_ = DBuf(dev_, stride_ * opt_.batch + 8);
    rawArena_ = DBuf(dev_, rawStride_ * opt_.batch + 8);
    dev_->sync();  // stream-ordered allocation made on the null stream: publish it to the plan's streams
    for (int s = 0; s < usedStreams_; s++) { void *h; check(evab_stream_create(dev_->ctx(), &h)); streams_.push_back(h); }
    for (int e = 0; e < numEvents_ + usedStreams_ + 1; e++) { void *h; check(evab_event_create(dev_->ctx(), &h)); events_.push_back(h); }
    // plan-time constants: raw values and (optionally) their encodings
    evalRawAndEncodes(nullptr);
    rawDirty_ = false;
    // galois tables for every rotation in the program
    for (auto &st : steps_)
      if ((st.op == Op::RotateLeftConst || st.op == Op::RotateRightConst) && *st.term->rotation != 0) {
        const u64 elt = galoisElt(*st.term);
        if (!keys_.galois.count(elt)) throw std::invalid_argument("Galois key not present");
        check(evab_galois_prepare(dev_->ctx(), elt));
        // shared mod-up: the key-dependent constant of (element, level), computed once per plan
        if (opt_.hoistModUp && st.hoist >= 0) {
          const int ell = vals_[st.term->index].ell;
          auto key = std::make_pair(elt, ell);
          if (!hoistConst_.count(key)) {
            DBuf cadd(dev_, evab_hoist_const_bytes(dev_->ctx(), ell) / 8), tmp(dev_, (std::size_t)(ell + 1) * N_);
            check(evab_rotate_hoist_const(dev_->ctx(), ell, elt, keys_.galois.at(elt).get(), cadd.get(), tmp.get(), nullptr));
            dev_->sync();
            hoistConst_.emplace(key, std::move(cadd));
          }
        }
      }
    hoistNeedsC0_.assign(hoistSrc.size(), 0);
    for (auto &ch : chunks_) hoistNeedsC0_[ch.gid] = 1;
    for (auto &Lz : lazy_) hoistNeedsC0_[Lz.gid] = 1;
    for (auto &ch : chunks_)
      for (const Term *r : ch.rots) {
        const u64 elt = galoisElt(*r);
        if (!keys_.galois.count(elt)) throw std::invalid_argument("Galois key not present");
        check(evab_galois_prepare(dev_->ctx(), elt));
        auto key = std::make_pair(elt, ch.ell);
        if (!hoistConst_.count(key)) {
          DBuf cadd(dev_, evab_hoist_const_bytes(dev_->ctx(), ch.ell) / 8), tmp(dev_, (std::size_t)(ch.ell + 1) * N_);
          check(evab_rotate_hoist_const(dev_->ctx(), ch.ell, elt, keys_.galois.at(elt).get(), cadd.get(), tmp.get(), nullptr));
          dev_->sync();
          hoistConst_.emplace(key, std::move(cadd));
        }
      }
    for (auto &Lz : lazy_)
      for (const Term *r : Lz.rots) {
        const u64 elt = galoisElt(*r);
        if (!keys_.galois.count(elt)) throw std::invalid_argument("Galois key not present");
        check(evab_galois_prepare(dev_->ctx(), elt));
        auto key = std::make_pair(elt, Lz.ell);
        if (!hoistConst_.count(key)) {
          DBuf cadd(dev_, evab_hoist_const_bytes(dev_->ctx(), Lz.ell) / 8), tmp(dev_, (std::size_t)(Lz.ell + 1) * N_);
          check(evab_rotate_hoist_const(dev_->ctx(), Lz.ell, elt, keys_.galois.at(elt).get(), cadd.get(), tmp.get(), nullptr));
          dev_->sync();
          hoistConst_.emplace(key, std::move(cadd));
        }
      }
    if (numFlags_) check(evab_host_alloc(8 * numFlags_ * 8 * (std::size_t)opt_.batch, (void **)&hostFlags_));
  }
  // Packed arena: describes every region of the plan to packArena (one buffer per materialised value; one per rotation chunk,
  // lazy rotation sum, encode group and hoist group covering all their members), then moves every offset to the packed
  // layout and adds the write-after-read waits it asks for.  Steps, launches and their operands' values are unchanged.
  template <class StepOperands>
  void packLayout(const std::vector<const Term *> &hoistSrc, const std::vector<std::size_t> &workWords, StepOperands stepOperands) {
    const std::uint64_t TC = prog_.termCount();
    const std::size_t H = hoistSrc.size(), L = lazy_.size();
    const int nSteps = (int)steps_.size();
    std::unordered_map<std::uint64_t, int> stepOf;   // producer -> step
    std::vector<int> stepOfEvent(numEvents_, -1);
    for (int i = 0; i < nSteps; i++) {
      stepOf[steps_[i].producer] = i;
      if (steps_[i].record >= 0) stepOfEvent[steps_[i].record] = i;
    }
    std::vector<PackStep> ps(nSteps);
    for (int i = 0; i < nSteps; i++) {
      ps[i].stream = steps_[i].stream;
      for (int e : steps_[i].waits) if (stepOfEvent[e] >= 0) ps[i].waits.push_back(stepOfEvent[e]);
    }
    std::vector<PackBuffer> pb;
    auto newBuf = [&](std::size_t words, int writer, bool pinned) {
      pb.push_back(PackBuffer{(words + 63) & ~std::size_t(63), writer, {}, pinned});   // 512-byte aligned, like the unpacked stride
      return (int)pb.size() - 1;
    };
    auto writerOf = [&](std::uint64_t producer) { auto f = stepOf.find(producer); return f == stepOf.end() ? -1 : f->second; };
    std::vector<int> bufOfVal(TC, -1), hoistBuf(H, -1), lazyBuf(L, -1), chunkBuf(chunks_.size(), -1), groupBuf(groups_.size(), -1);
    for (auto &t : order_) {
      const ValueInfo &v = vals_[t->index];
      if ((v.kind != Kind::Cipher && v.kind != Kind::Plain) || v.alias || v.fused || t->op == Op::Encode || chunkOf_.count(t->index) ||
          directOf_.count(t->index))
        continue;
      const std::size_t words = (std::size_t)(v.kind == Kind::Cipher ? v.size : 1) * v.ell * N_;
      bufOfVal[t->index] = t->op == Op::Input ? newBuf(words, 0, true) : newBuf(words, stepOf.at(t->index), false);
    }
    auto extWords = [&](int ell) { return opt_.hoistModUp ? evab_rotate_modup_ext_bytes(dev_->ctx(), ell) / 8 : 0; };
    for (std::size_t g = 0; g < H; g++) {
      const int ell = vals_[hoistSrc[g]->index].ell;
      if (int w = writerOf(TC + g); w >= 0) hoistBuf[g] = newBuf((std::size_t)ell * N_ + extWords(ell), w, false);
    }
    for (std::size_t l = 0; l < L; l++) lazyBuf[l] = newBuf(lazy_[l].roots.size() * 2 * (std::size_t)lazy_[l].ell * N_, stepOf.at(TC + H + l), false);
    for (std::size_t c = 0; c < chunks_.size(); c++) chunkBuf[c] = newBuf(chunks_[c].rots.size() * 2 * (std::size_t)chunks_[c].ell * N_, stepOf.at(TC + H + L + c), false);
    auto groupPlainWords = [&](const EncodeGroup &g) { return (std::size_t)(g.ell + (g.withP ? 1 : 0)) * N_; };
    for (std::size_t g = 0; g < groups_.size(); g++) {
      const EncodeGroup &G = groups_[g];
      const std::size_t words = G.members.size() * groupPlainWords(G) + evab_encode_work_bytes(dev_->ctx(), (int)G.members.size() - G.nUniform) / 8;
      groupBuf[g] = newBuf(words, stepOf.at(G.first->index), !G.dynamic && opt_.cacheConstants);   // cached constants: encoded at plan time
    }
    const int flagsBuf = numFlags_ ? newBuf(8 * numFlags_, 0, true) : -1;
    std::vector<int> workBuf(usedStreams_);
    for (int s = 0; s < usedStreams_; s++) workBuf[s] = newBuf(workWords[s], 0, true);
    // storage of a term: aliases (Output, duplicate terms) resolve to their source; chunk members and encode members to their composite
    auto bufOfTerm = [&](std::uint64_t x) -> int {
      while (vals_[x].alias) x = aliasSource(byIndex_[x]);
      if (vals_[x].kind != Kind::Cipher && vals_[x].kind != Kind::Plain) return -1;
      if (auto c = chunkOf_.find(x); c != chunkOf_.end()) return chunkBuf[c->second];
      if (auto d = directOf_.find(x); d != directOf_.end()) return lazyBuf[d->second.first];
      if (byIndex_[x]->op == Op::Encode) return groupBuf[groupIndex_.at(x)];
      return bufOfVal[x];
    };
    auto read = [&](int step, int b) { if (b >= 0) pb[b].readers.push_back(step); };
    for (int i = 0; i < nSteps; i++) {
      const Step &st = steps_[i];
      const std::uint64_t src = st.term->index;
      if (st.op == Op::Undef) {   // pseudo steps (hoist, rotation chunk, lazy rotation sums) read the group's source
        read(i, bufOfTerm(src));
        if (st.chunk >= 0) read(i, hoistBuf[chunks_[st.chunk].gid]);
        if (st.lazy >= 0) {
          read(i, hoistBuf[lazy_[st.lazy].gid]);
          for (auto &ws : lazy_[st.lazy].wts) for (const Term *w : ws) if (w) read(i, bufOfTerm(w->index));
          for (auto &ws : lazy_[st.lazy].twts) for (const Term *w : ws) if (w) read(i, bufOfTerm(w->index));
          for (const Term *x : lazy_[st.lazy].taps) read(i, bufOfTerm(x->index));
        }
        continue;
      }
      for (const Term *o : stepOperands(st.term)) read(i, bufOfTerm(o->index));   // a fused sum reads its leaves
      if (auto lz = lazyOfRoot_.find(src); lz != lazyOfRoot_.end()) for (auto &lo : lz->second) read(i, lazyBuf[lo.first]);
      if (st.hoist >= 0) read(i, hoistBuf[st.hoist]);
    }
    for (auto &o : prog_.getOutputs()) if (int b = bufOfTerm(o.second->index); b >= 0) pb[b].pinned = true;   // downloaded after the run

    const PackResult pr = packArena(ps, pb);
    auto at = [&](int b) { return pr.offsets.at(b); };
    for (auto &t : order_) if (bufOfVal[t->index] >= 0) vals_[t->index].off = at(bufOfVal[t->index]);
    for (std::size_t g = 0; g < H; g++)
      if (hoistBuf[g] >= 0) {
        hoistOff_[g] = at(hoistBuf[g]);
        if (opt_.hoistModUp) hoistExtOff_[g] = hoistOff_[g] + (std::size_t)vals_[hoistSrc[g]->index].ell * N_;
      }
    for (std::size_t l = 0; l < L; l++) lazy_[l].tempOff = at(lazyBuf[l]);
    for (auto &kv : directOf_) vals_[kv.first].off = lazy_[kv.second.first].tempOff + (std::size_t)kv.second.second * 2 * lazy_[kv.second.first].ell * N_;
    for (std::size_t c = 0; c < chunks_.size(); c++) {
      RotChunk &ch = chunks_[c];
      ch.outOff = at(chunkBuf[c]);
      for (std::size_t i = 0; i < ch.rots.size(); i++) vals_[ch.rots[i]->index].off = ch.outOff + i * 2 * (std::size_t)ch.ell * N_;
    }
    for (std::size_t g = 0; g < groups_.size(); g++) {
      EncodeGroup &G = groups_[g];
      G.outOff = at(groupBuf[g]);
      for (std::size_t i = 0; i < G.members.size(); i++) vals_[G.members[i]->index].off = G.outOff + i * groupPlainWords(G);
      G.workOff = G.outOff + G.members.size() * groupPlainWords(G);
    }
    for (auto &kv : encodeAlias_) vals_[kv.first].off = vals_[kv.second->index].off;
    if (flagsBuf >= 0) flagsOff_ = at(flagsBuf);
    for (int s = 0; s < usedStreams_; s++) workOff_[s] = at(workBuf[s]);
    for (auto &t : order_) if (vals_[t->index].alias) vals_[t->index].off = vals_[aliasSource(t)].off;
    for (auto &st : steps_) {
      if (st.lazyTemps.empty()) continue;
      st.lazyTemps.clear();
      for (auto &lo : lazyOfRoot_.at(st.term->index)) st.lazyTemps.push_back(lazy_[lo.first].tempOff + (std::size_t)lo.second * 2 * lazy_[lo.first].ell * N_);
    }
    for (auto &w : pr.waits) {   // write-after-read edges: the reusing step waits on the event of the last reader
      Step &last = steps_[w.second];
      if (last.record < 0) last.record = numEvents_++;
      std::vector<int> &waits = steps_[w.first].waits;
      if (std::find(waits.begin(), waits.end(), last.record) == waits.end()) waits.push_back(last.record);
    }
    reuseWaits_ = (long)pr.waits.size();
    keptAfterRun_.assign(TC, 0);
    for (auto &t : order_) if (int b = bufOfTerm(t->index); b >= 0) keptAfterRun_[t->index] = pb[b].pinned;
    stride_ = (pr.peak + 63) & ~std::size_t(63);
    packed_ = true;
  }
  // canonical (first) occurrence of a term that repeats an earlier one (dedupTerms)
  const Term *C(const Term *t) const { return byIndex_[canon_[t->index]]; }
  std::uint64_t aliasSource(const Term *t) const { return canon_[t->index] != t->index ? canon_[t->index] : t->operandAt(0)->index; }
  int levelToEll(std::uint32_t level) const {
    const int ell = k_ - 1 - (int)level;
    if (ell < 1) throw std::runtime_error("level exceeds the modulus chain");
    return ell;
  }
  u64 galoisElt(const Term &t) const {
    const int steps = t.op == Op::RotateLeftConst ? *t.rotation : -*t.rotation;
    const u64 elt = evab_galois_elt_from_step(N_, steps);
    if (!elt) throw std::invalid_argument("step count too large");
    return elt;
  }

  // raw (vector<double>) terms run on the host (reference seal_executor.h:63-112);
  // Encode terms whose operand does not depend on raw inputs are encoded once.
  void evalRawAndEncodes(void *stream) {
    hasDynamicEncodes_ = false;
    std::vector<char> dyn(prog_.termCount(), 0);
    for (int b = 0; b < opt_.batch; b++) {
      auto &raws = rawsB_[b];
      for (auto &t : order_) {
        const ValueInfo &v = vals_[t->index];
        bool d = (t->op == Op::Input && v.kind == Kind::Raw);
        for (auto &o : t->getOperands()) d = d || dyn[o->index];
        dyn[t->index] = d;
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
          if (encodeAlias_.count(t->index)) continue;
          auto &x = raws[t->operandAt(0)->index];
          if (x.empty()) continue;
          if (dyn[t->index]) hasDynamicEncodes_ = true;
          const std::uint64_t key = t->index * 65536ull + (std::uint64_t)b;
          if (!rawUploaded_.count(key) || dyn[t->index]) {
            if ((N_ / 2) % x.size()) throw std::runtime_error("Vector size must exactly divide the slot count");
            dev_->upload(rawArena_.get() + (std::size_t)b * rawStride_ + rawOff_.at(t->index), x.data(), x.size() * 8, stream);
            rawUploaded_.insert(key);
          }
        }
      }
    }
    dev_->sync(stream);  // the staged host vectors must outlive the copies
    if (opt_.cacheConstants && !staticEncoded_) {
      BatchGuard bg(opt_.batch, stride_, rawStride_);
      for (auto &g : groups_) if (!g.dynamic) issueEncodeGroup(g, stream);
      dev_->sync(stream);
      staticEncoded_ = true;
    }
  }
  // one batched device encode (scatter -> inverse FFT -> round/reduce -> NTT) for a group
  void issueEncodeGroup(const EncodeGroup &g, void *stream) {
    if (g.nUniform) {   // replicated scalars: constant polynomials, no FFT / NTT needed (bit-identical)
      std::vector<double> v, sc;
      for (int i = 0; i < g.nUniform; i++) { v.push_back(rawsB_[0][g.members[i]->operandAt(0)->index][0]); sc.push_back(vals_[g.members[i]->index].scale); }
      check(evab_encode_uniform_ext(dev_->ctx(), g.nUniform, v.data(), sc.data(), g.ell, g.withP ? 1 : 0, arena_.get() + g.outOff, stream));
    }
    const int rest = (int)g.members.size() - g.nUniform;
    if (!rest) return;
    std::vector<const double *> ptrs; std::vector<std::uint32_t> vec; std::vector<double> sc;
    for (int i = g.nUniform; i < (int)g.members.size(); i++) {
      Term *t = g.members[i];
      ptrs.push_back(reinterpret_cast<const double *>(rawArena_.get() + rawOff_.at(t->index)));
      vec.push_back((std::uint32_t)rawsB_[0][t->operandAt(0)->index].size());
      sc.push_back(vals_[t->index].scale);
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
    TraceScope(const Step &st, bool print, bool nvtx_) : nvtx(nvtx_) {
      if (!print && !nvtx) return;
      char name[96];
      const Term &t = *st.term;
      const char *pseudo = st.chunk >= 0 ? "RotationBatch" : st.lazy >= 0 ? "LazyRotationSums" : "InverseNTT";   // pseudo steps: named after their source term
      if (st.op == Op::Undef) std::snprintf(name, sizeof(name), "t%lu.%s", (unsigned long)t.index, pseudo);
      else std::snprintf(name, sizeof(name), "t%lu %s%s", (unsigned long)t.index, opName(t.op), st.sum.empty() ? "" : "(fused sum)");
      if (print) {
        std::printf("EVA: Execute t%lu%s = %s(", (unsigned long)t.index, st.op == Op::Undef ? "'" : "", st.op == Op::Undef ? pseudo : opName(t.op));
        bool first = true;
        if (st.op == Op::Undef) std::printf("t%lu", (unsigned long)t.index);
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
    const Term &t = *st.term;
    TraceScope trace(st, verbosity() >= 2, traceNvtx());
    evab_ctx *c = dev_->ctx();
    const ValueInfo &o = vals_[t.index];
    u64 *out = arena_.get() + o.off;
    if (st.chunk >= 0) {   // up to 16 rotations of one ciphertext, three launches
      const RotChunk &ch = chunks_[st.chunk];
      if (verbosity() >= 2)
        for (const Term *r : ch.rots)
          std::printf("EVA: Execute t%lu = %s(t%lu)  [stream %d, in the batch above]\n", (unsigned long)r->index, opName(r->op), (unsigned long)r->operandAt(0)->index, st.stream);
      std::vector<u64> elts; std::vector<const u64 *> keys, cadds;
      for (const Term *r : ch.rots) {
        const u64 elt = galoisElt(*r);
        elts.push_back(elt); keys.push_back(keys_.galois.at(elt).get());
        cadds.push_back(hoistConst_.at(std::make_pair(elt, ch.ell)).get());
      }
      check(evab_rotate_modup_many(c, ch.ell, (int)elts.size(), arena_.get() + ch.outOff, arena_.get() + o.off, arena_.get() + hoistExtOff_[ch.gid], elts.data(),
                                   keys.data(), cadds.data(), arena_.get() + workOff_[st.stream], stream));
      return;
    }
    if (st.lazy >= 0) {   // out_o = sum_i w_oi (.) rotate(x, g_i): approxHoist, one mod-down per sum; rotationSums, exact (+ taps)
      const LazySum &Lz = lazy_[st.lazy];
      std::vector<u64> elts; std::vector<const u64 *> keys, cadds, wts, taps, twts;
      for (const Term *r : Lz.rots) {
        const u64 elt = galoisElt(*r);
        elts.push_back(elt); keys.push_back(keys_.galois.at(elt).get());
        cadds.push_back(hoistConst_.at(std::make_pair(elt, Lz.ell)).get());
      }
      for (auto &ws : Lz.wts) for (const Term *w : ws) wts.push_back(w ? arena_.get() + vals_[w->index].off : nullptr);
      if (!opt_.approxHoist) {
        for (const Term *x : Lz.taps) taps.push_back(arena_.get() + vals_[x->index].off);
        for (auto &ws : Lz.twts) for (const Term *w : ws) twts.push_back(w ? arena_.get() + vals_[w->index].off : nullptr);
        check(evab_rotate_wsum(c, Lz.ell, (int)Lz.roots.size(), arena_.get() + Lz.tempOff, arena_.get() + o.off, arena_.get() + hoistExtOff_[Lz.gid], (int)elts.size(),
                               elts.data(), keys.data(), cadds.data(), wts.data(), (int)taps.size(), taps.data(), twts.data(), arena_.get() + workOff_[st.stream], stream));
        return;
      }
      check(evab_lazy_rotsum(c, Lz.ell, (int)Lz.roots.size(), arena_.get() + Lz.tempOff, arena_.get() + o.off, arena_.get() + hoistExtOff_[Lz.gid], (int)elts.size(),
                             elts.data(), keys.data(), cadds.data(), wts.data(), arena_.get() + workOff_[st.stream], stream));
      return;
    }
    if (st.op == Op::Undef) {   // shared inverse NTT of a rotation group's input
      if (opt_.hoistModUp)
      {
        check(evab_rotate_modup_prepare(c, o.ell, arena_.get() + hoistOff_[st.hoist], arena_.get() + hoistExtOff_[st.hoist], arena_.get() + o.off,
                                        arena_.get() + flagsOff_ + 8 * (std::size_t)st.hoist, stream));
        if (hoistNeedsC0_[st.hoist]) check(evab_rotate_modup_scale_c0(c, o.ell, arena_.get() + hoistExtOff_[st.hoist], arena_.get() + o.off, stream));
      }
      else
        check(evab_rotate_prepare(c, o.ell, arena_.get() + hoistOff_[st.hoist], arena_.get() + o.off, stream));
      return;
    }
    if (!st.sum.empty() || !st.lazyTemps.empty()) {   // fused multiply_plain / add tree
      std::vector<const u64 *> cts, pts; std::vector<int> sizes;
      for (auto &l : st.sum) {
        cts.push_back(arena_.get() + vals_[l.first->index].off);
        sizes.push_back(vals_[l.first->index].size);
        pts.push_back(l.second ? arena_.get() + vals_[l.second->index].off : nullptr);
      }
      std::vector<int> kinds = st.sumKind;
      for (std::size_t off : st.lazyTemps) { cts.push_back(arena_.get() + off); sizes.push_back(2); pts.push_back(nullptr); kinds.push_back(0); }
      check(evab_sum_products(c, o.ell, out, (int)cts.size(), cts.data(), sizes.data(), pts.data(), kinds.data(), stream));
      return;
    }
    auto V = [&](int i) -> const ValueInfo & { return vals_[t.operandAt(i)->index]; };
    auto P = [&](int i) -> const u64 * { return arena_.get() + vals_[t.operandAt(i)->index].off; };
    u64 *work = arena_.get() + workOff_[st.stream];
    switch (t.op) {
      case Op::Encode: {
        const EncodeGroup &g = groups_[groupIndex_.at(t.index)];
        if (g.first == &t && (g.dynamic || !opt_.cacheConstants)) issueEncodeGroup(g, stream);
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
          if (st.hoist >= 0 && opt_.hoistModUp)
            check(evab_rotate_modup_prepared(c, o.ell, out, P(0), arena_.get() + hoistExtOff_[st.hoist], elt, keys_.galois.at(elt).get(),
                                             hoistConst_.at(std::make_pair(elt, o.ell)).get(), work, stream));
          else if (st.hoist >= 0) check(evab_rotate_prepared(c, o.ell, out, P(0), arena_.get() + hoistOff_[st.hoist], elt, keys_.galois.at(elt).get(), work, stream));
          else check(evab_rotate(c, o.ell, out, P(0), elt, keys_.galois.at(elt).get(), work, stream));
        }
        break;
      case Op::Relinearize: check(evab_relinearize(c, o.ell, out, P(0), keys_.relin.get(), work, stream)); break;
      case Op::ModSwitch: check(evab_mod_switch(c, V(0).ell, out, P(0), V(0).size, stream)); break;
      case Op::Rescale: check(evab_rescale(c, V(0).ell, out, P(0), V(0).size, work, stream)); break;
      default: throw std::runtime_error(std::string("Unhandled op ") + opName(t.op));
    }
  }
  // fork from `stream` into the plan's streams, issue every step, join back
  void replay(void *stream) {
    evab_ctx *c = dev_->ctx();
    BatchGuard bg(opt_.batch, stride_, rawStride_);
    void *forkEv = events_[numEvents_ + usedStreams_];
    for (int b = 0; numFlags_ && b < opt_.batch; b++)   // zero-coefficient flags of the shared mod-ups
      check(evab_memset_zero(c, arena_.get() + (std::size_t)b * stride_ + flagsOff_, 8 * numFlags_ * 8, stream));
    check(evab_event_record(c, forkEv, stream));
    for (int s = 0; s < usedStreams_; s++) check(evab_stream_wait_event(c, streams_[s], forkEv));
    for (auto &st : steps_) {
      void *s = streams_[st.stream];
      for (int e : st.waits) check(evab_stream_wait_event(c, s, events_[e]));
      issue(st, s);
      if (st.record >= 0) check(evab_event_record(c, events_[st.record], s));
    }
    for (int s = 0; s < usedStreams_; s++) {
      check(evab_event_record(c, events_[numEvents_ + s], streams_[s]));
      check(evab_stream_wait_event(c, stream, events_[numEvents_ + s]));
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
  CkksEncoder &enc_;
  const KeySet &keys_;
  Program &prog_;
  ExecOptions opt_;
  u64 N_;
  int k_;
  std::vector<Term *> order_;
  std::vector<Term *> byIndex_;          // term index -> term
  std::vector<std::uint64_t> canon_;     // term index -> index of the first identical term (itself when unique)
  std::vector<ValueInfo> vals_;
  std::vector<std::vector<std::vector<double>>> rawsB_;   // [instance][term]
  std::size_t stride_ = 0, rawStride_ = 0;
  std::vector<EncodeGroup> groups_;
  std::vector<Term *> encodeTerms_;
  std::unordered_map<std::uint64_t, int> groupIndex_;
  std::unordered_map<std::uint64_t, std::size_t> rawOff_;
  std::vector<std::size_t> hoistOff_;   // arena word offset of every hoist buffer
  std::vector<char> hoistNeedsC0_;                           // hoist group feeds evab_rotate_modup_many / evab_lazy_rotsum
  std::vector<RotChunk> chunks_;                             // rotationChunk
  std::unordered_map<std::uint64_t, int> chunkOf_;
  std::vector<LazySum> lazy_;                                // approxHoist
  std::unordered_map<std::uint64_t, std::vector<std::pair<int, int>>> lazyOfRoot_;   // fused sum -> (lazy sum, output)
  std::unordered_map<std::uint64_t, std::pair<int, int>> directOf_;   // rotationSums: fused sum stored as (lazy sum, output) itself
  std::set<std::uint64_t> needP_;                            // Encode terms whose plaintext carries the extra row mod P
  std::vector<std::size_t> hoistExtOff_;                     // ... and of the group's extended digits (hoistModUp)
  std::size_t flagsOff_ = 0, numFlags_ = 0;                  // zero-coefficient flags, 8 words apart
  std::map<std::pair<u64, int>, DBuf> hoistConst_;           // (galois element, ell) -> cadd [2][ell+1][N]
  u64 *hostFlags_ = nullptr;                                 // page-locked copy of the flags of the last run
  std::unordered_map<std::uint64_t, Term *> encodeAlias_;  // Encode term -> identical earlier Encode term
  std::unordered_set<std::uint64_t> rawUploaded_;
  std::size_t rawWords_ = 0;
  bool staticEncoded_ = false;
  DBuf rawArena_;
  std::vector<Step> steps_;
  std::unordered_map<std::uint64_t, int> recordAfter_;
  std::unordered_set<std::uint64_t> encoded_;
  std::vector<std::size_t> workOff_;
  std::vector<void *> streams_, events_;
  void *capStream_ = nullptr;
  void *mainStream_ = nullptr;
  void *graph_ = nullptr;
  bool graphValid_ = false, rawDirty_ = false, rawInputs_ = false, hasDynamicEncodes_ = false;
  int numEvents_ = 0, usedStreams_ = 0;
  std::size_t cipherOps_ = 0;
  bool packed_ = false;                  // arena laid out by packArena (storage of dead values reused)
  std::size_t unpackedBytes_ = 0;        // arenaBytes() of the one-offset-per-value layout
  long reuseWaits_ = 0;                  // event waits packArena added
  std::vector<char> keptAfterRun_;       // packed plan: term index -> its storage is pinned (inputs, outputs, cached constants)
  DBuf arena_;
};

}  // namespace evab
