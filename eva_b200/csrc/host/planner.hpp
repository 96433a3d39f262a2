// planner.hpp -- lowers a compiled EVA program ONCE into a static plan: value kinds, levels, scales, the plan-level
// rewrites (fused sums, rotation groups, rotation sums, rotation chunks, encode groups), the stream and event schedule and
// the arena layout.  Pure host code: no device calls, so that plans can be built and checked without a GPU
// (tests/test_planner.py).  executor.hpp materialises a Plan on the device and replays it.
#pragma once
#include "../host_tables.hpp"
#include "arena_packer.hpp"
#include "ir.hpp"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <set>
#include <tuple>
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

// Term: one program term.  The other kinds are pseudo steps, named after the source ciphertext of their hoist group:
// Hoist computes the group's shared inverse NTT (and mod-up), RotationChunk up to 16 of its rotations, RotationSum
// one evab_rotate_wsum / evab_lazy_rotsum call
enum class StepKind { Term, Hoist, RotationChunk, RotationSum };

struct Step {
  StepKind kind = StepKind::Term;
  const Term *term = nullptr;  // Term: the term it issues; pseudo steps: the source ciphertext of their hoist group
  int stream = 0;
  std::vector<int> waits;  // event ids to wait for before issuing
  int record = -1;         // event id recorded after issuing
  // fused sum (root Add of a tree of cipher+cipher Adds): out = sum of ct (* pt when pt != null)
  std::vector<std::pair<const Term *, const Term *>> sum;
  std::vector<int> sumKind;    // per leaf: 0 ciphertext, 1 ciphertext * plaintext, 2 ciphertext (x) ciphertext
  std::vector<std::pair<int, int>> rotSums;  // fused sum: (rotation sum, output) added to the other leaves
  int hoist = -1;              // the hoist group whose shared buffers this step reads
  int index = -1;              // pseudo steps: the hoist group, rotation chunk or rotation sum the step computes
  std::uint64_t producer = 0;  // term index; termCount + group, + rotation sum or + chunk for pseudo steps
};

// Encode terms of one level that are encoded by a single batched device launch sequence
struct EncodeGroup {
  int ell; bool dynamic; std::vector<Term *> members; std::size_t outOff = 0, workOff = 0; int stream = -1;
  Term *first = nullptr;   // earliest member in program order: its step issues the whole group
  int nUniform = 0;        // leading members whose vector is a replicated scalar: one-pass encoder
  bool withP = false;      // plaintexts of this group carry an extra residue row mod the key-switch prime (approxHoist)
};

// rotationChunk: up to 16 rotations of one hoist group computed by one evab_rotate_modup_many call (3 launches instead of 3 n)
struct RotChunk {
  int gid = 0, ell = 0;
  std::vector<const Term *> rots;
  std::size_t outOff = 0;                           // their results, contiguous: [n][2][ell][N]
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
  bool allStatic = true;
};

// One block of the arena: a value, a composite (hoist group, rotation sum outputs, rotation chunk, encode group with its
// workspace), the zero-digit flags or a stream's workspace.  Both layouts are laid out from this one table.
struct Region {
  std::size_t words = 0;
  int writer = -1;            // the step that writes it; -1: not written by a run (pinned), or never materialised (not pinned)
  std::vector<int> readers;   // the steps that read it
  bool pinned = false;        // inputs, outputs, cached constants, flags, workspaces: never reused
  std::size_t off = 0;        // word offset
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

// Scratch bytes of the device calls a plan issues: the C-ABI's evab_*_bytes, filled in by the Executor from its context
struct WorkSizes {
  std::function<std::size_t(int ell)> keyswitch, rotateModupExt;
  std::function<std::size_t(int size)> rescale;
  std::function<std::size_t(int ell, int n)> rotateModupMany;
  std::function<std::size_t(int ell, int n, int nout)> rotateWsum;
  std::function<std::size_t(int ell, int nout)> lazyRotsum;
  std::function<std::size_t(int count)> encode;
};

struct Plan {
  ExecOptions opt;
  std::uint64_t N = 0;
  std::uint64_t terms = 0;                      // term indices: the program's terms, then the plan's own rotation hops
  std::vector<Term *> order;                    // the program's terms (and hops) in topological order
  std::vector<Term *> byIndex;                  // term index -> term
  std::vector<std::uint64_t> canon;             // term index -> index of the first identical term (itself when unique)
  std::vector<ValueInfo> vals;
  std::vector<std::vector<double>> constants;   // term index -> the expanded vector of a Constant term (empty otherwise)
  std::vector<char> dyn;                        // term index -> depends on a raw input
  std::size_t cipherOps = 0;
  // composeRotations: rotations whose step has no Galois key run as chains of rotations by NAF terms.  The intermediate hops are
  // terms of the plan (RotateLeftConst by the term's signed step, no operands, indices from the program's termCount()); their
  // storage is a program of their own, never the user's
  std::unique_ptr<Program> hopProgram;
  std::vector<Term::Ptr> hops;
  std::unordered_map<std::uint64_t, const Term *> chainSrc;   // hop or composed rotation -> the ciphertext it rotates
  std::unordered_map<std::uint64_t, int> lastHop;             // composed rotation of the program -> the step of its last hop
  std::map<std::uint64_t, std::vector<int>> chain;            // every key-switched rotation of the program -> the steps it applies
  long composedRotations = 0;
  std::vector<const Term *> hoistSrc;           // hoist group -> the ciphertext its rotations read
  std::vector<std::size_t> hoistOff, hoistExtOff;   // arena word offsets of every hoist buffer and of its extended digits (hoistModUp)
  std::vector<char> needsC0;                    // hoist group feeds evab_rotate_modup_many / evab_lazy_rotsum
  std::vector<RotChunk> chunks;                 // rotationChunk
  std::unordered_map<std::uint64_t, int> chunkOf;
  std::vector<LazySum> lazy;                    // approxHoist / rotationSums
  std::unordered_map<std::uint64_t, std::vector<std::pair<int, int>>> lazyOfRoot;   // fused sum -> (rotation sum, output)
  std::unordered_map<std::uint64_t, std::pair<int, int>> directOf;   // rotationSums: fused sum stored as (rotation sum, output) itself
  std::set<std::uint64_t> needP;                // Encode terms whose plaintext carries the extra row mod P
  std::vector<EncodeGroup> groups;
  std::unordered_map<std::uint64_t, int> groupIndex;
  std::unordered_map<std::uint64_t, Term *> encodeAlias;   // Encode term -> identical earlier Encode term
  std::unordered_map<std::uint64_t, std::size_t> rawOff;   // Encode term -> word offset of its staged vector in the raw arena
  std::size_t rawWords = 0;
  std::size_t flagsOff = 0, numFlags = 0;       // zero-coefficient flags, 8 words apart
  std::vector<Step> steps;
  int numEvents = 0, usedStreams = 0;
  std::vector<std::size_t> workOff;             // per stream
  std::size_t stride = 0, rawStride = 0;        // words per instance
  std::vector<Region> regions;
  std::vector<int> storage;                     // term index -> the region holding its value (-1: none)
  bool packed = false;                          // arena laid out by packArena (storage of dead values reused)
  std::size_t unpackedBytes = 0;                // arenaBytes() of the one-offset-per-value layout
  long reuseWaits = 0;                          // event waits packArena added

  std::size_t arenaBytes() const { return (stride * (std::size_t)opt.batch + 8 + rawStride * (std::size_t)opt.batch + 8) * 8; }
  // words a region takes in this plan's layout: packed regions are 512-byte aligned, like the unpacked stride
  std::size_t laidWords(const Region &r) const { return !packed ? r.words : r.writer < 0 && !r.pinned ? 0 : (r.words + 63) & ~std::size_t(63); }
  std::size_t rotSumOff(std::pair<int, int> lo) const { const LazySum &L = lazy[lo.first]; return L.tempOff + (std::size_t)lo.second * 2 * L.ell * N; }
  // canonical (first) occurrence of a term that repeats an earlier one (dedupTerms)
  const Term *C(const Term *t) const { return byIndex[canon[t->index]]; }
  std::uint64_t aliasSource(const Term *t) const { return canon[t->index] != t->index ? canon[t->index] : t->operandAt(0)->index; }
  // the ciphertext a rotation reads: its operand, or the previous hop of its chain
  const Term *src(const Term *r) const { auto f = chainSrc.find(r->index); return f != chainSrc.end() ? f->second : C(r->operandAt(0).get()); }
  // the step a rotation applies (SEAL's rotate_vector argument): its own, or the last hop's of its chain
  int stepOf(const Term *r) const {
    if (auto f = lastHop.find(r->index); f != lastHop.end()) return f->second;
    return r->op == Op::RotateLeftConst ? *r->rotation : -*r->rotation;
  }
  // every rotation the plan issues, and whether it uses a shared mod-up (and so the hoist constant of its (element, ell))
  template <class F> void forEachRotation(F f) const {
    for (auto &st : steps)
      if (st.kind == StepKind::Term && (st.term->op == Op::RotateLeftConst || st.term->op == Op::RotateRightConst) && *st.term->rotation != 0)
        f(st.term, opt.hoistModUp && st.hoist >= 0);
    for (auto &ch : chunks) for (const Term *r : ch.rots) f(r, true);
    for (auto &L : lazy) for (const Term *r : L.rots) f(r, true);
  }

  // shape of the plan (test / tooling hook)
  std::map<std::string, long> planStats() const {
    std::map<std::string, long> m;
    m["steps"] = (long)steps.size(); m["streams"] = usedStreams; m["hoist_groups"] = (long)hoistSrc.size();
    m["rotation_chunks"] = (long)chunks.size(); m["chunked_rotations"] = 0;
    const bool approx = opt.approxHoist;   // lazy holds the approximate (lazy_*) or the exact (rotation_sum_*) calls
    m["lazy_calls"] = approx ? (long)lazy.size() : 0; m["rotation_sum_calls"] = approx ? 0 : (long)lazy.size();
    m["lazy_sums"] = m["lazy_rotations"] = m["rotation_sums"] = m["rotation_sum_rotations"] = m["rotation_sum_taps"] = 0;
    for (auto &L : lazy) {
      m[approx ? "lazy_sums" : "rotation_sums"] += (long)L.roots.size();
      m[approx ? "lazy_rotations" : "rotation_sum_rotations"] += (long)L.rots.size();
      m["rotation_sum_taps"] += (long)L.taps.size();
    }
    for (auto &c : chunks) m["chunked_rotations"] += (long)c.rots.size();
    long elided = 0;
    for (auto &t : order) if ((t->op == Op::RotateLeftConst || t->op == Op::RotateRightConst) && vals[t->index].fused) elided++;
    m["elided_rotations"] = elided;
    m["composed_rotations"] = composedRotations; m["composed_hops"] = (long)hops.size();
    m["arena_bytes"] = (long)arenaBytes(); m["arena_bytes_unpacked"] = (long)unpackedBytes; m["packed"] = packed ? 1 : 0;
    m["reuse_waits"] = reuseWaits;
    long constWords = 0;   // plaintexts of plan-time constants, resident for the plan's lifetime
    if (opt.cacheConstants)
      for (auto &g : groups) if (!g.dynamic) constWords += (long)g.members.size() * (g.ell + (g.withP ? 1 : 0)) * (long)N;
    m["constant_bytes"] = constWords * 8 * opt.batch;
    return m;
  }
};

// The passes, run in this order by buildPlan (below).  Each reads what the earlier ones derived.
class Planner {
public:
  // galoisElements: the Galois elements that have keys (null: every step has its own)
  Planner(Program &prog, const ExecOptions &opt, std::uint64_t N, int k, const WorkSizes &ws, const std::set<std::uint64_t> *galoisElements)
      : prog_(prog), ws_(ws), k_(k), elts_(galoisElements) {
    p.opt = opt;
    p.N = N;
  }
  Plan run(std::size_t arenaLimit) {
    inferValues();
    composeRotations();
    fuseSums();
    groupRotations();
    sumRotations();
    chunkRotations();
    groupEncodes();
    schedule();
    layout(arenaLimit);
    return std::move(p);
  }

private:
  // ---- 1. value kinds, sizes, levels and scales (SEAL's error conditions); duplicate terms alias their first occurrence
  void inferValues() {
    const ExecOptions &opt = p.opt;
    for (auto &t : prog_.toposort()) p.order.push_back(t.get());  // raw: the plan lives inside the Program (attachment)
    const std::uint64_t TC = p.terms = prog_.termCount();
    p.vals.assign(TC, ValueInfo{});
    if (opt.batch < 1) throw std::invalid_argument("batch must be >= 1");
    p.constants.assign(TC, {});
    p.byIndex.assign(TC, nullptr);
    p.canon.resize(TC);
    for (std::size_t i = 0; i < TC; i++) p.canon[i] = i;
    std::map<std::tuple<int, long long, std::uint64_t, std::uint64_t>, std::uint64_t> seenTerm;
    for (auto &t : p.order) {
      ValueInfo &v = p.vals[t->index];
      p.byIndex[t->index] = t;
      auto a = [&](int i) -> const ValueInfo & { return p.vals[t->operandAt(i)->index]; };
      if (opt.dedupTerms && t->numOperands() >= 1 && p.vals[t->operandAt(0)->index].kind != Kind::Raw &&
          (t->op == Op::Add || t->op == Op::Sub || t->op == Op::Mul || t->op == Op::Negate || t->op == Op::RotateLeftConst ||
           t->op == Op::RotateRightConst || t->op == Op::Relinearize || t->op == Op::ModSwitch || t->op == Op::Rescale)) {
        const long long attr = t->rotation ? (long long)*t->rotation : (t->rescaleDivisor ? (long long)*t->rescaleDivisor : 0);
        const std::uint64_t o0 = p.canon[t->operandAt(0)->index], o1 = t->numOperands() > 1 ? p.canon[t->operandAt(1)->index] : ~0ull;
        auto ins = seenTerm.emplace(std::make_tuple((int)t->op, attr, o0, o1), t->index);
        if (!ins.second && p.vals[ins.first->second].kind == Kind::Cipher) {
          p.canon[t->index] = ins.first->second;
          v = p.vals[ins.first->second]; v.alias = true;     // same value: shares the first occurrence's storage
          p.cipherOps++;                                     // still an executed IR term of the program
          continue;
        }
      }
      switch (t->op) {
        case Op::Input: {
          const Type ty = t->type.value_or(Type::Cipher);
          if (ty == Type::Raw) { v.kind = Kind::Raw; break; }
          if (!t->encodeAtScale || !t->encodeAtLevel) throw std::runtime_error("input term lacks scale/level (program not compiled?)");
          v.kind = ty == Type::Cipher ? Kind::Cipher : Kind::Plain;
          v.size = 2; v.ell = levelToEll(*t->encodeAtLevel); v.scale = std::ldexp(1.0, (int)*t->encodeAtScale);
          if (v.kind == Kind::Cipher && !opt.inputSizes.empty())
            for (auto &in : prog_.getInputs())
              if (in.second.get() == t) { auto f = opt.inputSizes.find(in.first); if (f != opt.inputSizes.end()) v.size = f->second; }
          if (v.size < 2 || v.size > 3) throw std::runtime_error("input ciphertext size must be 2 or 3");
        } break;
        case Op::Constant:
          v.kind = Kind::Raw;
          t->constant->expandTo(p.constants[t->index], prog_.getVecSize());
          break;
        case Op::Encode:
          if (a(0).kind != Kind::Raw) throw std::runtime_error("Encode expects a raw operand");
          v.kind = Kind::Plain; v.ell = levelToEll(t->encodeAtLevel.value()); v.scale = std::ldexp(1.0, (int)t->encodeAtScale.value());
          encodeTerms_.push_back(t);
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
        } break;
        case Op::Negate:
          if (a(0).kind == Kind::Raw) { v.kind = Kind::Raw; break; }
          v = a(0); v.alias = false;
          break;
        case Op::RotateLeftConst: case Op::RotateRightConst:
          if (a(0).kind == Kind::Raw) { v.kind = Kind::Raw; break; }
          if (a(0).kind != Kind::Cipher || a(0).size != 2) throw std::runtime_error("rotation expects a size-2 ciphertext");
          v = a(0); v.alias = false;
          break;
        case Op::Relinearize:
          if (a(0).kind != Kind::Cipher) throw std::runtime_error("Relinearize expects a ciphertext");
          v = a(0); v.alias = false; v.size = 2;
          break;
        case Op::ModSwitch: case Op::Rescale:
          if (a(0).kind != Kind::Cipher) throw std::runtime_error("ModSwitch/Rescale expects a ciphertext");
          if (a(0).ell < 2) throw std::invalid_argument("end of modulus switching chain reached");
          v = a(0); v.alias = false; v.ell = a(0).ell - 1;
          if (t->op == Op::Rescale) v.scale = a(0).scale / std::ldexp(1.0, (int)t->rescaleDivisor.value());
          break;
        case Op::Output:
          v = a(0); v.alias = true;
          break;
        default: throw std::runtime_error(std::string("Unhandled op ") + opName(t->op));
      }
      if (v.kind == Kind::Cipher && t->op != Op::Input && t->op != Op::Output) p.cipherOps++;
    }
  }

  // ---- 1b. composed rotations (SEAL 3.6 Evaluator::rotate_internal): a ciphertext rotation whose step has no Galois key is the chain
  // of rotations by the NAF terms of its step (evab_host::rotation_hops), each an ordinary key switch.  The chains of one source
  // share their prefixes, a trie keyed by Galois elements.  A prefix node is a plan-owned hop, or the value of a program rotation
  // of the same source that computes exactly it: a rotation by its single term, or a keyless rotation whose own chain it is (a
  // longer prefix whose sum has a key of its own is a different value).  The last hop of a chain is the program's term itself.
  // Later passes see ordinary rotations: Plan::src and Plan::stepOf give what each reads and applies.  Without composed rotations
  // the plan is unchanged.
  void composeRotations() {
    const std::uint64_t N = p.N;
    auto has = [&](std::uint64_t e) { return !elts_ || elts_->count(e) > 0; };
    std::vector<Term *> rots;
    for (Term *t : p.order)
      if ((t->op == Op::RotateLeftConst || t->op == Op::RotateRightConst) && *t->rotation != 0 && p.vals[t->index].kind == Kind::Cipher &&
          p.canon[t->index] == t->index && evab_host::galois_elt_from_step(N, p.stepOf(t)))   // (a step too large: the executor's error)
        rots.push_back(t);
    // (source, Galois elements of the chain) -> the term holding that value; program rotations first, in program order
    std::map<std::pair<std::uint64_t, std::vector<std::uint64_t>>, const Term *> node;
    auto eltsOf = [&](const std::vector<int> &steps, std::size_t n) {
      std::vector<std::uint64_t> e;
      for (std::size_t j = 0; j < n; j++) e.push_back(evab_host::galois_elt_from_step(N, steps[j]));
      return e;
    };
    for (Term *t : rots) {
      std::vector<int> &hops = p.chain[t->index] = evab_host::rotation_hops(N, p.stepOf(t), has);
      node.emplace(std::make_pair(p.src(t)->index, eltsOf(hops, hops.size())), t);
    }
    for (Term *t : rots) {
      const int s = p.stepOf(t);
      const std::vector<int> hops = p.chain.at(t->index);
      if (has(evab_host::galois_elt_from_step(N, s))) continue;
      const Term *prev = p.src(t);
      const std::uint64_t x = prev->index;
      for (std::size_t j = 1; j < hops.size(); j++) {
        auto key = std::make_pair(x, eltsOf(hops, j));
        auto f = node.find(key);
        if (f == node.end()) {   // a plan-owned hop
          if (!p.hopProgram) p.hopProgram = std::make_unique<Program>("rotation hops", prog_.getVecSize());
          Term::Ptr h = p.hopProgram->makeTerm(Op::RotateLeftConst);
          h->rotation = hops[j - 1];
          h->index = p.terms++;
          ValueInfo v = p.vals[t->index];
          v.alias = v.fused = false;
          p.vals.push_back(v); p.canon.push_back(h->index); p.byIndex.push_back(h.get()); p.constants.emplace_back();
          p.chainSrc[h->index] = prev;
          p.hops.push_back(h);
          f = node.emplace(std::move(key), h.get()).first;
        }
        prev = f->second;
      }
      p.chainSrc[t->index] = prev;
      p.lastHop[t->index] = hops.back();
      p.composedRotations++;
    }
    if (!p.composedRotations) return;
    // every hop and every prefix value before its first reader (the sources of the chains come before them already)
    std::vector<Term *> order;
    std::vector<char> placed(p.terms, 0);
    std::function<void(Term *)> place = [&](Term *t) {
      if (placed[t->index]) return;
      placed[t->index] = 1;
      if (auto f = p.chainSrc.find(t->index); f != p.chainSrc.end()) place(p.byIndex[f->second->index]);
      order.push_back(t);
    };
    for (Term *t : p.order) place(t);
    p.order = std::move(order);
  }

  // ---- 2. fused sums: a tree of cipher+cipher Adds whose inner nodes have a single use collapses into
  // one kernel; leaves that are single-use multiply_plain results are multiplied on the fly
  // (Sobel / Harris filter taps: sum_i rot_i(x) * w_i).  Same canonical result, see evab_sum_terms.
  void fuseSums() {
    if (!p.opt.fuseSums) return;
    std::vector<int> uses = useCounts();
    auto isCipherAdd = [&](const Term *t) {
      return t->op == Op::Add && p.vals[t->operandAt(0)->index].kind == Kind::Cipher && p.vals[t->operandAt(1)->index].kind == Kind::Cipher;
    };
    auto plainMul = [&](const Term *t, const Term *&ct, const Term *&pt) {
      if (t->op != Op::Mul) return false;
      const Term *a = p.C(t->operandAt(0).get()), *b = p.C(t->operandAt(1).get());
      if (p.vals[a->index].kind == Kind::Cipher && p.vals[b->index].kind == Kind::Plain) { ct = a; pt = b; return true; }
      if (p.vals[b->index].kind == Kind::Cipher && p.vals[a->index].kind == Kind::Plain) { ct = b; pt = a; return true; }
      return false;
    };
    // Evaluator::multiply / square of two size-2 ciphertexts (2x2 -> 3)
    auto cipherMul = [&](const Term *t, const Term *&a, const Term *&b) {
      if (t->op != Op::Mul) return false;
      a = p.C(t->operandAt(0).get()); b = p.C(t->operandAt(1).get());
      return p.vals[a->index].kind == Kind::Cipher && p.vals[b->index].kind == Kind::Cipher && p.vals[a->index].size == 2 && p.vals[b->index].size == 2;
    };
    for (auto it = p.order.rbegin(); it != p.order.rend(); ++it) {
      Term *root = *it;
      if (!isCipherAdd(root) || p.vals[root->index].fused || p.vals[root->index].alias) continue;
      std::vector<std::pair<const Term *, const Term *>> leaves;
      std::vector<int> kinds;
      std::vector<const Term *> absorbed;
      std::function<void(const Term *)> expand = [&](const Term *t) {
        const Term *ct = nullptr, *pt = nullptr;
        const bool inner = t != root;
        if ((!inner || uses[t->index] == 1) && isCipherAdd(t) && leaves.size() + 2 <= 30) {
          if (inner) absorbed.push_back(t);
          expand(p.C(t->operandAt(0).get()));
          expand(p.C(t->operandAt(1).get()));
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
      for (const Term *t : absorbed) p.vals[t->index].fused = true;
      sumOf_[root->index] = std::move(leaves);
      sumKindOf_[root->index] = std::move(kinds);
    }
  }

  // ---- 3. hoisted rotations: two or more rotations of the same ciphertext share the inverse NTT of
  // its c1 (evab_rotate_prepare); the shared buffer is produced by a pseudo step of its own
  void groupRotations() {
    if (!p.opt.hoistRotations) return;
    std::map<std::uint64_t, std::vector<const Term *>> bySrc;
    for (auto &t : p.order)
      if ((t->op == Op::RotateLeftConst || t->op == Op::RotateRightConst) && *t->rotation != 0 && p.vals[t->index].kind == Kind::Cipher &&
          p.vals[t->index].ell <= 15 && !p.vals[t->index].alias)
        bySrc[p.src(t)->index].push_back(t);
    for (auto &kv : bySrc) {
      if (kv.second.size() < 2) continue;
      const int gid = (int)p.hoistSrc.size();
      p.hoistSrc.push_back(p.src(kv.second.front()));
      for (const Term *r : kv.second) hoistOf_[r->index] = gid;
    }
    if (p.opt.hoistModUp) p.numFlags = p.hoistSrc.size();   // one zero-coefficient flag per group
  }

  // ---- 4. rotation sums.  approxHoist (opt-in): leaves "rotation of a hoist group (x) constant plaintext" of a fused sum, two or more
  // of the same group, become ONE lazy rotation sum whose temporary joins the remaining leaves; a rotation all of whose uses went that
  // way is never materialised.  The plaintexts involved are encoded with an extra residue row mod P.
  // rotationSums (exact, evab_rotate_wsum): the same grouping, for rotations whose every use is such a leaf with a scalar constant
  // weight.  A leaf of weight 0.0 is dropped (its product is the zero ciphertext), and the sum's other leaves "size-2 ciphertext
  // (x) scalar constant" join the call as taps (a rotation by 0 through its operand).  A sum left with no other leaf is the call's
  // output itself: it is never issued as a step of its own.
  void sumRotations() {
    const ExecOptions &opt = p.opt;
    const bool exactSums = !opt.approxHoist && opt.rotationSums;
    if (!((opt.approxHoist || exactSums) && opt.hoistModUp && opt.fuseSums)) return;
    const std::uint64_t TC = p.terms;
    std::vector<int> usesAll = useCounts(), lazyUses(TC, 0), wsumLeaves(TC, 0), pos(TC, 0);
    for (std::size_t i = 0; i < p.order.size(); i++) pos[p.order[i]->index] = (int)i;
    std::set<const Term *> chainRead;   // rotations that a hop of a composed rotation reads
    for (auto &kv : p.chainSrc) chainRead.insert(kv.second);
    auto scalarWeight = [&](const Term *pt, double &v) {
      if (pt->op != Op::Encode || pt->operandAt(0)->op != Op::Constant || !replicatedScalar(pt)) return false;
      v = p.constants[pt->operandAt(0)->index][0];
      return true;
    };
    auto rotLeaf = [&](const std::pair<const Term *, const Term *> &l) {
      double v;
      return hoistOf_.count(l.first->index) && p.vals[l.first->index].size == 2 && (exactSums ? scalarWeight(l.second, v) : l.second->op == Op::Encode);
    };
    if (exactSums)
      for (auto &kv : sumOf_)
        for (std::size_t i = 0; i < kv.second.size(); i++)
          if (sumKindOf_.at(kv.first)[i] == 1 && rotLeaf(kv.second[i])) wsumLeaves[kv.second[i].first->index]++;
    std::map<int, int> openOf;   // hoist group -> the lazy sum that still takes outputs
    for (auto &t : p.order) {
      auto f = sumOf_.find(t->index);
      if (f == sumOf_.end()) continue;
      auto &leaves = f->second;
      auto &kinds = sumKindOf_.at(t->index);
      std::map<int, std::vector<int>> byGroup;
      for (int i = 0; i < (int)leaves.size(); i++) {
        if (kinds[i] != 1 || !rotLeaf(leaves[i])) continue;
        if (exactSums && wsumLeaves[leaves[i].first->index] != usesAll[leaves[i].first->index]) continue;
        if (chainRead.count(leaves[i].first)) continue;   // materialised for the hops that read it: used as it is
        byGroup[hoistOf_.at(leaves[i].first->index)].push_back(i);
      }
      auto isZero = [&](int i) { double v = 1.0; return exactSums && scalarWeight(leaves[i].second, v) && v == 0.0; };
      std::vector<char> drop(leaves.size(), 0);
      std::vector<std::pair<int, std::vector<int>>> slices;   // at most 16 rotations per call: longer sums are cut
      for (auto &kv : byGroup)
        for (std::size_t b = 0; b < kv.second.size(); b += 16)
          slices.emplace_back(kv.first, std::vector<int>(kv.second.begin() + b, kv.second.begin() + std::min(kv.second.size(), b + 16)));
      std::vector<int> zeroSlices;   // leaves of slices whose weights are all 0.0: dropped when the sum takes a rotation sum call
      for (auto &kv : slices) {
        if (std::all_of(kv.second.begin(), kv.second.end(), isZero)) { zeroSlices.insert(zeroSlices.end(), kv.second.begin(), kv.second.end()); continue; }
        if (kv.second.size() < 2) continue;
        // sums over rotations of the same ciphertext share one call (and the inner products of the rotations they have in
        // common), as long as the later sum's weights are available when the first one runs
        int li = -1;
        if (auto op = openOf.find(kv.first); op != openOf.end()) {
          LazySum &L = p.lazy[op->second];
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
          li = (int)p.lazy.size();
          p.lazy.emplace_back();
          p.lazy[li].gid = kv.first; p.lazy[li].ell = p.vals[t->index].ell;
          openOf[kv.first] = li;
        }
        LazySum &L = p.lazy[li];
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
          if (!exactSums) p.needP.insert(leaves[i].second->index);
        }
        p.lazyOfRoot[t->index].emplace_back(li, (int)L.roots.size() - 1);
      }
      if (!p.lazyOfRoot.count(t->index)) continue;
      for (int i : zeroSlices) { drop[i] = 1; lazyUses[leaves[i].first->index]++; }
      if (exactSums) {   // the other scalar-weighted leaves: taps of the first call, when they are computed before that call is issued
        const auto [li, o] = p.lazyOfRoot.at(t->index).front();
        LazySum &L = p.lazy[li];
        for (int i = 0; i < (int)leaves.size(); i++) {
          double v;
          if (drop[i] || kinds[i] != 1 || p.vals[leaves[i].first->index].size != 2 || !scalarWeight(leaves[i].second, v)) continue;
          const Term *ct = leaves[i].first;
          const bool rot0 = (ct->op == Op::RotateLeftConst || ct->op == Op::RotateRightConst) && *ct->rotation == 0;
          const Term *src = rot0 ? p.C(ct->operandAt(0).get()) : ct;
          if (p.vals[src->index].fused || pos[src->index] >= pos[L.roots.front()->index]) continue;
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
      if (exactSums && leaves.empty() && p.lazyOfRoot.at(t->index).size() == 1) p.directOf[t->index] = p.lazyOfRoot.at(t->index).front();
    }
    for (auto &t : p.order)
      if (lazyUses[t->index] && lazyUses[t->index] == usesAll[t->index]) p.vals[t->index].fused = true;   // the rotation is never materialised
  }

  // ---- 5. batched rotations: the (materialised) rotations of a hoist group are computed together, 16 per call
  void chunkRotations() {
    if (p.opt.rotationChunk >= 2 && p.opt.hoistModUp) {
      std::vector<int> open(p.hoistSrc.size(), -1);
      for (auto &t : p.order) {
        auto h = hoistOf_.find(t->index);
        if (h == hoistOf_.end() || p.vals[t->index].fused || p.canon[t->index] != t->index) continue;
        int ci = open[h->second];
        if (ci < 0 || (int)p.chunks[ci].rots.size() >= std::min(16, p.opt.rotationChunk)) {
          ci = open[h->second] = (int)p.chunks.size();
          p.chunks.emplace_back();
          p.chunks[ci].gid = h->second; p.chunks[ci].ell = p.vals[t->index].ell;
        }
        p.chunkOf[t->index] = ci;
        p.chunks[ci].rots.push_back(t);
      }
    }
    p.needsC0.assign(p.hoistSrc.size(), 0);
    for (auto &ch : p.chunks) p.needsC0[ch.gid] = 1;
    if (p.opt.approxHoist)   // evab_lazy_rotsum reads P * c0 on ext's diagonal; evab_rotate_wsum reads c0 itself
      for (auto &L : p.lazy) p.needsC0[L.gid] = 1;
  }

  // ---- 6. Encode groups: one batched device encode per (ell, input-dependent?) group.
  // Static groups (constants only) are encoded once per plan when cacheConstants is
  // set, otherwise every run like the reference (seal_executor.h:303-308).
  void groupEncodes() {
    p.dyn.assign(p.terms, 0);
    for (auto &t : p.order) {
      bool d = (t->op == Op::Input && p.vals[t->index].kind == Kind::Raw);
      for (auto &o : t->getOperands()) d = d || p.dyn[o->index];
      p.dyn[t->index] = d;
    }
    std::map<std::tuple<int, int, int>, int> groupOf;
    // identical constant vectors encoded at the same level and scale give identical plaintexts:
    // later occurrences alias the first one (same bits as encoding each, seal_executor.h:217-248)
    std::map<std::tuple<int, double, std::vector<double>, int>, Term *> firstOf;
    for (Term *t : encodeTerms_) {
      if (p.opt.dedupConstants && !p.dyn[t->index] && t->operandAt(0)->op == Op::Constant) {
        auto ck = std::make_tuple(p.vals[t->index].ell, p.vals[t->index].scale, p.constants[t->operandAt(0)->index], (int)p.needP.count(t->index));
        auto ins = firstOf.emplace(std::move(ck), t);
        if (!ins.second) {
          p.encodeAlias[t->index] = ins.first->second;
          p.groupIndex[t->index] = p.groupIndex.at(ins.first->second->index);
          continue;
        }
      }
      auto key = std::make_tuple(p.vals[t->index].ell, (int)p.dyn[t->index], (int)p.needP.count(t->index));
      auto it = groupOf.find(key);
      if (it == groupOf.end()) {
        it = groupOf.emplace(key, (int)p.groups.size()).first;
        p.groups.push_back(EncodeGroup{std::get<0>(key), std::get<1>(key) != 0, {}});
        p.groups.back().withP = std::get<2>(key) != 0;
      }
      p.groups[it->second].members.push_back(t);
      p.groupIndex[t->index] = it->second;
    }
    for (auto &g : p.groups) {
      g.first = g.members.front();
      if (!g.dynamic && p.opt.uniformEncode) {   // scalar constants first: they go through evab_encode_uniform
        auto mid = std::stable_partition(g.members.begin(), g.members.end(), [&](Term *t) { return replicatedScalar(t); });
        g.nUniform = (int)(mid - g.members.begin());
      }
      for (Term *t : g.members) { p.rawOff[t->index] = p.rawWords; p.rawWords += prog_.getVecSize(); }
    }
  }

  // ---- 7. stream assignment + event edges.  Producers are identified by term index, or termCount + hoist group,
  // + rotation sum, + chunk for the pseudo steps.
  void schedule() {
    const std::uint64_t TC = p.terms, H = p.hoistSrc.size(), L = p.lazy.size();
    const int S = std::max(1, p.opt.numStreams);
    const std::size_t NP = TC + H + L + p.chunks.size();
    std::unordered_map<std::uint64_t, std::uint64_t> prodOf;   // rotation term -> the chunk step that produces it
    std::unordered_map<std::uint64_t, int> recordAfter;
    std::vector<int> streamOf(NP, -1), eventOf(NP, -1);
    std::vector<char> chainTaken(NP, 0), inputTerm(NP, 0), emitted(NP, 0);
    workWords_.assign(S, 0);
    int rr = 0;
    for (auto &t : p.order) if (t->op == Op::Input) inputTerm[t->index] = 1;
    // place one step: continue the chain of a device operand nobody continued yet, else take a new
    // stream round-robin; cross-stream operands become event waits
    auto emit = [&](Step st, std::vector<std::uint64_t> operands, int forced, std::size_t w) {
      for (auto &o : operands) if (auto f = prodOf.find(o); f != prodOf.end()) o = f->second;
      int chosen = forced;
      for (std::uint64_t o : operands) {
        const int so = streamOf[o];
        if (so >= 0 && !chainTaken[o] && !inputTerm[o]) { chosen = so; chainTaken[o] = 1; break; }
      }
      if (chosen < 0) chosen = (rr++) % S;
      st.stream = chosen;
      for (std::uint64_t o : operands) {
        const int so = streamOf[o];
        if (so >= 0 && so != chosen && !inputTerm[o]) {
          if (eventOf[o] < 0) { eventOf[o] = p.numEvents++; recordAfter[o] = eventOf[o]; }
          if (std::find(st.waits.begin(), st.waits.end(), eventOf[o]) == st.waits.end()) st.waits.push_back(eventOf[o]);
        }
      }
      workWords_[chosen] = std::max(workWords_[chosen], w);
      streamOf[st.producer] = chosen;
      p.steps.push_back(st);
    };
    // pseudo steps are emitted once, before their first consumer; the hoist step of their group goes first
    auto pseudo = [&](StepKind kind, int index, int gid, std::uint64_t producer) {
      Step s;
      s.kind = kind; s.term = p.hoistSrc[gid]; s.index = index; s.producer = producer;
      if (kind != StepKind::Hoist) s.hoist = gid;
      return s;
    };
    auto emitHoist = [&](int gid) {
      if (emitted[TC + gid]) return;
      emitted[TC + gid] = 1;
      emit(pseudo(StepKind::Hoist, gid, gid, TC + gid), {p.hoistSrc[gid]->index}, -1, 0);
    };
    auto emitRotSum = [&](int li) {
      const LazySum &Lz = p.lazy[li];
      const std::uint64_t id = TC + H + (std::size_t)li;
      if (emitted[id]) return id;
      emitted[id] = 1;
      emitHoist(Lz.gid);
      std::vector<std::uint64_t> ops{p.hoistSrc[Lz.gid]->index, TC + (std::uint64_t)Lz.gid};
      for (auto &ws : Lz.wts) for (const Term *w : ws) if (w && streamOf[w->index] >= 0) ops.push_back(w->index);   // (later sums' constants: same encode group)
      for (auto &ws : Lz.twts) for (const Term *w : ws) if (w && streamOf[w->index] >= 0) ops.push_back(w->index);
      for (const Term *x : Lz.taps) ops.push_back(x->index);
      const bool exact = !p.opt.approxHoist;
      const std::size_t work = exact ? ws_.rotateWsum(Lz.ell, (int)Lz.rots.size(), (int)Lz.roots.size()) : ws_.lazyRotsum(Lz.ell, (int)Lz.roots.size());
      emit(pseudo(StepKind::RotationSum, li, Lz.gid, id), ops, -1, work / 8);
      return id;
    };
    auto emitChunk = [&](int ci) {   // computed with the other rotations of its chunk
      const RotChunk &ch = p.chunks[ci];
      const std::uint64_t id = TC + H + L + (std::size_t)ci;
      if (emitted[id]) return;
      emitted[id] = 1;
      emitHoist(ch.gid);
      emit(pseudo(StepKind::RotationChunk, ci, ch.gid, id), {p.hoistSrc[ch.gid]->index, TC + (std::uint64_t)ch.gid}, -1,
           ws_.rotateModupMany(ch.ell, (int)ch.rots.size()) / 8);
      for (const Term *r : ch.rots) { prodOf[r->index] = id; streamOf[r->index] = streamOf[id]; }
    };
    for (auto &t : p.order) {
      const ValueInfo &v = p.vals[t->index];
      const bool device = (v.kind == Kind::Cipher || v.kind == Kind::Plain) && t->op != Op::Input && !v.alias && !v.fused;
      if (!device) {
        if (v.alias) streamOf[t->index] = streamOf[p.aliasSource(t)];
        continue;
      }
      if (auto d = p.directOf.find(t->index); d != p.directOf.end()) {   // the sum is a rotation sum call's output
        const std::uint64_t id = emitRotSum(d->second.first);
        prodOf[t->index] = id; streamOf[t->index] = streamOf[id];
        continue;
      }
      if (auto co = p.chunkOf.find(t->index); co != p.chunkOf.end()) { emitChunk(co->second); continue; }
      Step st;
      st.term = t; st.producer = t->index;
      if (auto f = sumOf_.find(t->index); f != sumOf_.end()) { st.sum = f->second; st.sumKind = sumKindOf_.at(t->index); }
      std::vector<std::uint64_t> operands;
      for (const Term *o : stepOperands(t)) operands.push_back(o->index);
      if (auto lz = p.lazyOfRoot.find(t->index); lz != p.lazyOfRoot.end())
        for (auto &lo : lz->second) {   // the rotation sums feeding this fused sum go first, as a pseudo step of their own
          operands.push_back(emitRotSum(lo.first));
          st.rotSums.push_back(lo);
        }
      int forced = -1;
      if (t->op == Op::Encode) {
        EncodeGroup &g = p.groups[p.groupIndex.at(t->index)];
        if (g.stream < 0) g.stream = (rr++) % S;
        forced = g.stream;
      }
      std::size_t w = 0;
      if (t->op == Op::Relinearize)
        w = ws_.keyswitch(p.vals[t->operandAt(0)->index].ell) / 8;
      else if ((t->op == Op::RotateLeftConst || t->op == Op::RotateRightConst) && *t->rotation != 0)
        w = ws_.keyswitch(p.vals[p.src(t)->index].ell) / 8;
      else if (t->op == Op::Rescale)
        w = ws_.rescale(p.vals[t->operandAt(0)->index].size) / 8;
      if (auto h = hoistOf_.find(t->index); h != hoistOf_.end()) {   // the group's shared inverse NTT goes first
        emitHoist(h->second);
        st.hoist = h->second;
        operands.push_back(TC + h->second);
      }
      emit(st, operands, forced, w);
    }
    for (auto &st : p.steps)
      if (auto it = recordAfter.find(st.producer); it != recordAfter.end()) st.record = it->second;
    // last step of every stream must be joined back into the caller's stream
    for (auto &st : p.steps) p.usedStreams = std::max(p.usedStreams, st.stream + 1);
  }

  // ---- 8. arena layout: every region of the table (regionTable) at its own offset when that fits the limit, else the storage
  // of dead values is reused (arena_packer.hpp); then the offsets of every value and composite member (placeMembers)
  void layout(std::size_t arenaLimit) {
    regionTable();
    std::size_t words = 0;
    for (auto &r : p.regions) { r.off = words; words += r.words; }
    p.stride = (words + 63) & ~std::size_t(63);
    p.rawStride = (p.rawWords + 7) & ~std::size_t(7);
    p.unpackedBytes = p.arenaBytes();
    if (p.unpackedBytes > arenaLimit) {
      pack();
      if (p.arenaBytes() > arenaLimit)
        throw std::runtime_error("plan arena needs " + std::to_string(p.arenaBytes()) + " bytes packed (" + std::to_string(p.unpackedBytes) +
                                 " bytes unpacked), more than the limit of " + std::to_string(arenaLimit) + " bytes");
    }
    placeMembers();
  }

  // Regions in layout order: values (those later absorbed into a fused sum, a chunk or a rotation sum output keep their words in
  // the one-offset-per-value layout, unwritten), hoist groups, rotation sums, chunks, encode groups, flags, workspaces
  void regionTable() {
    const std::uint64_t TC = p.terms, H = p.hoistSrc.size(), L = p.lazy.size();
    std::unordered_map<std::uint64_t, int> stepOf;   // producer -> step
    for (int i = 0; i < (int)p.steps.size(); i++) stepOf[p.steps[i].producer] = i;
    auto writerOf = [&](std::uint64_t producer) { auto f = stepOf.find(producer); return f == stepOf.end() ? -1 : f->second; };
    auto add = [&](std::size_t words, int writer, bool pinned) {
      p.regions.push_back(Region{words, writer, {}, pinned, 0});
      return (int)p.regions.size() - 1;
    };
    valR_.assign(TC, -1);
    for (auto &t : p.order) {
      const ValueInfo &v = p.vals[t->index];
      if ((v.kind != Kind::Cipher && v.kind != Kind::Plain) || v.alias || t->op == Op::Encode) continue;
      const bool own = !v.fused && !p.chunkOf.count(t->index) && !p.directOf.count(t->index);
      const bool input = t->op == Op::Input;
      valR_[t->index] = add((std::size_t)(v.kind == Kind::Cipher ? v.size : 1) * v.ell * p.N, own && !input ? stepOf.at(t->index) : -1, own && input);
    }
    hoistR_ = (int)p.regions.size();
    for (std::size_t g = 0; g < H; g++) {
      const int ell = p.vals[p.hoistSrc[g]->index].ell;
      add((std::size_t)ell * p.N + (p.opt.hoistModUp ? ws_.rotateModupExt(ell) / 8 : 0), writerOf(TC + g), false);
    }
    lazyR_ = (int)p.regions.size();
    for (std::size_t l = 0; l < L; l++) add(p.lazy[l].roots.size() * 2 * (std::size_t)p.lazy[l].ell * p.N, stepOf.at(TC + H + l), false);
    chunkR_ = (int)p.regions.size();
    for (std::size_t c = 0; c < p.chunks.size(); c++)
      add(p.chunks[c].rots.size() * 2 * (std::size_t)p.chunks[c].ell * p.N, stepOf.at(TC + H + L + c), false);
    groupR_ = (int)p.regions.size();
    for (auto &G : p.groups) {
      const bool cached = !G.dynamic && p.opt.cacheConstants;   // encoded at plan time
      add(G.members.size() * plainWords(G) + ws_.encode((int)G.members.size() - G.nUniform) / 8, cached ? -1 : stepOf.at(G.first->index), cached);
    }
    flagsR_ = p.numFlags ? add(8 * p.numFlags, -1, true) : -1;
    workR_ = (int)p.regions.size();
    for (int s = 0; s < p.usedStreams; s++) add(workWords_[s], -1, true);

    // storage of every term: aliases (Output, duplicate terms) resolve to their source; chunk members, rotation sum outputs and
    // encode members to their composite
    p.storage.assign(TC, -1);
    for (auto &t : p.order) {
      const std::uint64_t x = t->index;
      const ValueInfo &v = p.vals[x];
      int &s = p.storage[x];
      if (v.alias) s = p.storage[p.aliasSource(t)];
      else if (v.kind != Kind::Cipher && v.kind != Kind::Plain) s = -1;
      else if (auto c = p.chunkOf.find(x); c != p.chunkOf.end()) s = chunkR_ + c->second;
      else if (auto d = p.directOf.find(x); d != p.directOf.end()) s = lazyR_ + d->second.first;
      else if (t->op == Op::Encode) s = groupR_ + p.groupIndex.at(x);
      else s = v.fused ? -1 : valR_[x];
    }
    auto read = [&](int step, int r) { if (r >= 0) p.regions[r].readers.push_back(step); };
    for (int i = 0; i < (int)p.steps.size(); i++) {
      const Step &st = p.steps[i];
      if (st.kind == StepKind::Term) {
        for (const Term *o : stepOperands(st.term)) read(i, p.storage[o->index]);   // a fused sum reads its leaves
        for (auto &lo : st.rotSums) read(i, lazyR_ + lo.first);
      } else {
        read(i, p.storage[st.term->index]);   // pseudo steps read their group's source
      }
      if (st.kind == StepKind::RotationSum) {
        const LazySum &Lz = p.lazy[st.index];
        for (auto &ws : Lz.wts) for (const Term *w : ws) if (w) read(i, p.storage[w->index]);
        for (auto &ws : Lz.twts) for (const Term *w : ws) if (w) read(i, p.storage[w->index]);
        for (const Term *x : Lz.taps) read(i, p.storage[x->index]);
      }
      if (st.hoist >= 0) read(i, hoistR_ + st.hoist);
    }
    for (auto &o : prog_.getOutputs()) if (int r = p.storage[o.second->index]; r >= 0) p.regions[r].pinned = true;   // downloaded after the run
  }

  // packed layout: describes every region to packArena, takes its offsets and adds the write-after-read waits it asks for.
  // Steps, launches and their operands' values are unchanged.
  void pack() {
    p.packed = true;
    const int nSteps = (int)p.steps.size();
    std::vector<int> stepOfEvent(p.numEvents, -1);
    for (int i = 0; i < nSteps; i++) if (p.steps[i].record >= 0) stepOfEvent[p.steps[i].record] = i;
    std::vector<PackStep> ps(nSteps);
    for (int i = 0; i < nSteps; i++) {
      ps[i].stream = p.steps[i].stream;
      for (int e : p.steps[i].waits) if (stepOfEvent[e] >= 0) ps[i].waits.push_back(stepOfEvent[e]);
    }
    std::vector<PackBuffer> pb;
    for (auto &r : p.regions) pb.push_back(PackBuffer{p.laidWords(r), r.writer, r.readers, r.pinned});
    const PackResult pr = packArena(ps, pb);
    for (std::size_t r = 0; r < p.regions.size(); r++) p.regions[r].off = pr.offsets[r];
    for (auto &w : pr.waits) {   // write-after-read edges: the reusing step waits on the event of the last reader
      Step &last = p.steps[w.second];
      if (last.record < 0) last.record = p.numEvents++;
      std::vector<int> &waits = p.steps[w.first].waits;
      if (std::find(waits.begin(), waits.end(), last.record) == waits.end()) waits.push_back(last.record);
    }
    p.reuseWaits = (long)pr.waits.size();
    p.stride = (pr.peak + 63) & ~std::size_t(63);
  }

  // the one place where offsets of values and composite members are derived from their regions
  void placeMembers() {
    auto at = [&](int r) { return p.regions[r].off; };
    for (auto &t : p.order) if (valR_[t->index] >= 0) p.vals[t->index].off = at(valR_[t->index]);
    p.hoistOff.assign(p.hoistSrc.size(), 0);
    p.hoistExtOff.assign(p.hoistSrc.size(), 0);
    for (std::size_t g = 0; g < p.hoistSrc.size(); g++) {
      p.hoistOff[g] = at(hoistR_ + (int)g);
      p.hoistExtOff[g] = p.hoistOff[g] + (std::size_t)p.vals[p.hoistSrc[g]->index].ell * p.N;
    }
    for (std::size_t l = 0; l < p.lazy.size(); l++) p.lazy[l].tempOff = at(lazyR_ + (int)l);
    for (auto &kv : p.directOf) p.vals[kv.first].off = p.rotSumOff(kv.second);
    for (std::size_t c = 0; c < p.chunks.size(); c++) {
      RotChunk &ch = p.chunks[c];
      ch.outOff = at(chunkR_ + (int)c);
      for (std::size_t i = 0; i < ch.rots.size(); i++) p.vals[ch.rots[i]->index].off = ch.outOff + i * 2 * (std::size_t)ch.ell * p.N;
    }
    for (std::size_t g = 0; g < p.groups.size(); g++) {
      EncodeGroup &G = p.groups[g];
      G.outOff = at(groupR_ + (int)g);
      for (std::size_t i = 0; i < G.members.size(); i++) p.vals[G.members[i]->index].off = G.outOff + i * plainWords(G);
      G.workOff = G.outOff + G.members.size() * plainWords(G);
    }
    for (auto &kv : p.encodeAlias) p.vals[kv.first].off = p.vals[kv.second->index].off;
    if (flagsR_ >= 0) p.flagsOff = at(flagsR_);
    p.workOff.assign(p.usedStreams, 0);
    for (int s = 0; s < p.usedStreams; s++) p.workOff[s] = at(workR_ + s);
    // alias chains (Output of X shares X's storage; Output(Output) never occurs)
    for (auto &t : p.order) if (p.vals[t->index].alias) p.vals[t->index].off = p.vals[p.aliasSource(t)].off;
  }

  // uses of every canonical term by canonical terms
  std::vector<int> useCounts() const {
    std::vector<int> uses(p.terms, 0);
    for (auto &t : p.order) if (p.canon[t->index] == t->index) for (const Term *o : operands(t)) uses[o->index]++;
    return uses;
  }
  // the canonical terms a term reads (a rotation of a chain: the previous hop)
  std::vector<const Term *> operands(const Term *t) const {
    if (auto f = p.chainSrc.find(t->index); f != p.chainSrc.end()) return {f->second};
    std::vector<const Term *> ops;
    for (auto &o : t->getOperands()) ops.push_back(p.C(o.get()));
    return ops;
  }
  // the Encode term's vector is a replicated scalar (the uniform encoder's predicate)
  bool replicatedScalar(const Term *enc) const {
    const auto &x = p.constants[enc->operandAt(0)->index];
    return !x.empty() && std::all_of(x.begin(), x.end(), [&](double y) { return std::memcmp(&y, &x[0], sizeof(double)) == 0; });
  }
  // operands a step really reads (fused sums read their leaves)
  std::vector<const Term *> stepOperands(const Term *t) const {
    std::vector<const Term *> ops;
    auto f = sumOf_.find(t->index);
    if (f == sumOf_.end()) return operands(t);
    for (auto &l : f->second) { ops.push_back(l.first); if (l.second) ops.push_back(l.second); }
    return ops;
  }
  std::size_t plainWords(const EncodeGroup &g) const { return (std::size_t)(g.ell + (g.withP ? 1 : 0)) * p.N; }
  int levelToEll(std::uint32_t level) const {
    const int ell = k_ - 1 - (int)level;
    if (ell < 1) throw std::runtime_error("level exceeds the modulus chain");
    return ell;
  }

  Program &prog_;
  const WorkSizes &ws_;
  int k_;
  const std::set<std::uint64_t> *elts_;
  Plan p;
  std::vector<Term *> encodeTerms_;
  std::unordered_map<std::uint64_t, std::vector<std::pair<const Term *, const Term *>>> sumOf_;   // fused sum -> leaves
  std::unordered_map<std::uint64_t, std::vector<int>> sumKindOf_;
  std::unordered_map<std::uint64_t, int> hoistOf_;   // rotation term -> hoist group
  std::vector<std::size_t> workWords_;               // per stream
  std::vector<int> valR_;                            // term index -> its value's region (-1: none)
  int hoistR_ = 0, lazyR_ = 0, chunkR_ = 0, groupR_ = 0, flagsR_ = -1, workR_ = 0;   // first region of each kind
};

// N, k: the ring degree and the modulus count (with the key-switch prime); arenaLimit: bytes the arena may take
// galoisElements: the Galois elements that have keys; rotations by other steps are composed (null: every step has its own key)
inline Plan buildPlan(Program &program, const ExecOptions &opt, std::uint64_t N, int k, std::size_t arenaLimit, const WorkSizes &ws,
                      const std::set<std::uint64_t> *galoisElements = nullptr) {
  return Planner(program, opt, N, k, ws, galoisElements).run(arenaLimit);
}

}  // namespace evab
