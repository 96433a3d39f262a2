// compiler.hpp -- CKKS compiler for EVA programs (host side, no GPU work).
//
// Re-implementation of the reference compiler pipeline so that EVA scripts run
// unchanged against this backend (reference eva/ckks/ckks_compiler.h:36-306):
//   type deduction -> constant folding -> [reduction combining + log expansion]
//   -> rescaling policy {lazy_waterline (default), eager_waterline, always, minimum}
//   -> encode insertion -> {lazy, eager} relinearization -> modulus switching
//   (backward) -> lowering of plain - cipher -> validation (levels, parameters,
//   scales) -> encryption parameter / rotation key selection -> signature.
// Each pass below cites the reference header whose observable behaviour it
// reproduces; tests compare the output against programs compiled by the
// reference compiler itself (tests/golden/programs, built from /root/reference).
#pragma once
#include "backend.hpp"
#include <cstdarg>
#include <cstdio>
#include <numeric>
#include <unordered_map>

#include "logging.hpp"

namespace evab {

inline void warn(const char *fmt, ...) {
  va_list ap; va_start(ap, fmt);
  std::fprintf(stderr, "WARNING: "); std::vfprintf(stderr, fmt, ap); std::fprintf(stderr, "\n");
  va_end(ap);
}

// ---- configuration (reference eva/ckks/ckks_config.h:12-41, ckks_config.cpp:10-75) ----
enum class Rescaler { LazyWaterline, EagerWaterline, Always, Minimum };
struct CKKSConfig {
  bool balanceReductions = true;
  Rescaler rescaler = Rescaler::LazyWaterline;
  bool lazyRelinearize = true;
  std::uint32_t securityLevel = 128;
  bool quantumSafe = false;
  bool warnVecSize = true;

  CKKSConfig() {}
  explicit CKKSConfig(const std::unordered_map<std::string, std::string> &m) {
    // (no iostream parsing here: locale facets are unreliable inside extension modules)
    auto parseBool = [](const std::string &s, bool &out) {
      if (s == "true" || s == "True" || s == "1") { out = true; return true; }
      if (s == "false" || s == "False" || s == "0") { out = false; return true; }
      return false;
    };
    for (auto &e : m) {
      const std::string &k = e.first, &v = e.second;
      if (k == "balance_reductions") { if (!parseBool(v, balanceReductions)) warn("Could not parse boolean in balance_reductions=%s. Falling back to default.", v.c_str()); }
      else if (k == "rescaler") {
        if (v == "lazy_waterline") rescaler = Rescaler::LazyWaterline;
        else if (v == "eager_waterline") rescaler = Rescaler::EagerWaterline;
        else if (v == "always") rescaler = Rescaler::Always;
        else if (v == "minimum") rescaler = Rescaler::Minimum;
        else warn("Unknown value rescaler=%s. Available rescalers are lazy_waterline, eager_waterline, always, minimum. Falling back to default.", v.c_str());
      }
      else if (k == "lazy_relinearize") { if (!parseBool(v, lazyRelinearize)) warn("Could not parse boolean in lazy_relinearize=%s. Falling back to default.", v.c_str()); }
      else if (k == "security_level") {
        char *end = nullptr;
        unsigned long x = std::strtoul(v.c_str(), &end, 10);
        if (end == v.c_str() || *end) throw std::runtime_error("Could not parse unsigned int in security_level=" + v);
        securityLevel = (std::uint32_t)x;
      }
      else if (k == "quantum_safe") { if (!parseBool(v, quantumSafe)) throw std::runtime_error("Could not parse boolean in quantum_safe=" + v); }
      else if (k == "warn_vec_size") { if (!parseBool(v, warnVecSize)) warn("Could not parse boolean in warn_vec_size=%s. Falling back to default.", v.c_str()); }
      else warn("Unknown option %s. Available options are: balance_reductions, rescaler, lazy_relinearize, security_level, quantum_safe, warn_vec_size", k.c_str());
    }
  }
};

// HomomorphicEncryption.org standard: maximal total coeff-modulus bits per degree
// (classical / quantum-safe, 128/192/256-bit security); same tables SEAL ships.
inline int heStdMaxBits(std::uint32_t sec, bool quantum, std::size_t n) {
  static const int tc[3][6] = {{27, 54, 109, 218, 438, 881}, {19, 37, 75, 152, 305, 611}, {14, 29, 58, 118, 237, 476}};
  static const int tq[3][6] = {{25, 51, 101, 202, 411, 827}, {17, 35, 70, 141, 284, 571}, {13, 27, 54, 109, 220, 443}};
  int row = sec <= 128 ? 0 : sec <= 192 ? 1 : 2, col;
  switch (n) { case 1024: col = 0; break; case 2048: col = 1; break; case 4096: col = 2; break; case 8192: col = 3; break; case 16384: col = 4; break; case 32768: col = 5; break; default: return 0; }
  return quantum ? tq[row][col] : tc[row][col];
}

// optional side table
template <class T> class TermMapOpt : public TermMapBase {
public:
  explicit TermMapOpt(Program &p) : p_(p) { p_.registerMap(this); }
  ~TermMapOpt() override { p_.unregisterMap(this); }
  void resize(std::size_t n) override { if (v_.size() < n) v_.resize(n); }
  T &operator[](const Term::Ptr &t) { auto &o = v_.at(t->index); if (!o) o.emplace(); return *o; }
  T &at(const Term::Ptr &t) { return v_.at(t->index).value(); }
  bool has(const Term::Ptr &t) const { return v_.at(t->index).has_value(); }
private:
  Program &p_;
  std::vector<std::optional<T>> v_;
};

// Ready-stack traversal that tolerates rewrites around the current term
// (reference eva/common/program_traversal.h:36-88).
template <class F> void traverse(Program &program, bool forward, F &&rewrite) {
  TermMap<bool> ready(program), processed(program);
  std::vector<Term::Ptr> stack = forward ? program.getSources() : program.getSinks();
  for (auto &t : stack) ready[t] = 1;
  auto predsDone = [&](const Term::Ptr &t) {
    if (forward) { for (auto &o : t->getOperands()) if (!processed[o]) return false; }
    else { for (auto &u : t->getUses()) if (!processed[u]) return false; }
    return true;
  };
  std::vector<Term::Ptr> check;
  while (!stack.empty()) {
    Term::Ptr term = stack.back();
    stack.pop_back();
    check.clear();
    if (forward) { for (auto &s : term->getUses()) check.push_back(s); } else { for (auto &s : term->getOperands()) check.push_back(s); }
    rewrite(term);
    processed[term] = 1;
    for (auto &leaf : forward ? program.getSources() : program.getSinks())
      if (!ready[leaf]) { stack.push_back(leaf); ready[leaf] = 1; }
    if (forward) { for (auto &s : term->getUses()) check.push_back(s); } else { for (auto &s : term->getOperands()) check.push_back(s); }
    for (auto &s : check)
      if (!ready[s] && predsDone(s)) { stack.push_back(s); ready[s] = 1; }
  }
}

class CKKSCompiler {
public:
  CKKSCompiler() {}
  explicit CKKSCompiler(CKKSConfig c) : config_(c) {}
  explicit CKKSCompiler(const std::unordered_map<std::string, std::string> &m) : config_(m) {}

  std::tuple<std::unique_ptr<Program>, CKKSParameters, CKKSSignature> compile(Program &input) {
    auto program = input.deepCopy();
    Program &p = *program;
    TermMap<Type> types(p);
    TermMapOpt<std::uint32_t> scales(p);
    for (auto &src : p.getSources()) {
      if (!src->encodeAtScale) {
        for (auto &e : p.getInputs()) if (e.second == src) throw std::runtime_error("The scale for input " + e.first + " was not set.");
        throw std::runtime_error("The scale for a constant was not set.");
      }
      scales[src] = *src->encodeAtScale;
    }
    transform(p, types, scales);
    validate(p, types, scales);
    CKKSParameters params = selectParameters(p, types, scales);
    std::map<std::string, CKKSEncodingInfo> ins;
    for (auto &e : p.getInputs()) ins.emplace(e.first, CKKSEncodingInfo(e.second->type.value(), (int)e.second->encodeAtScale.value(), (int)e.second->encodeAtLevel.value()));
    return std::make_tuple(std::move(program), std::move(params), CKKSSignature((int)p.getVecSize(), std::move(ins)));
  }

private:
  typedef TermMap<Type> Types;
  typedef TermMapOpt<std::uint32_t> Scales;
  static bool isAddSub(Op o) { return o == Op::Add || o == Op::Sub; }
  static bool isRot(Op o) { return o == Op::RotateLeftConst || o == Op::RotateRightConst; }

  // ---- reference eva/common/type_deducer.h:19-37 ----
  static void deduceTypes(Program &p, Types &types) {
    traverse(p, true, [&](Term::Ptr &t) {
      if (t->numOperands() > 0) {
        Type inferred = Type::Raw;
        for (auto &o : t->getOperands()) if (types[o] == Type::Cipher) inferred = Type::Cipher;
        types[t] = t->op == Op::Encode ? Type::Plain : inferred;
      } else if (t->op == Op::Constant) types[t] = Type::Raw;
      else types[t] = t->type.value();
    });
  }

  // ---- reference eva/common/constant_folder.h:28-190: fold all-constant subtrees ----
  static void foldConstants(Program &p, Scales &scale) {
    const std::size_t vs = p.getVecSize();
    traverse(p, true, [&](Term::Ptr &t) {
      auto &args = t->getOperands();
      if (args.empty()) return;
      for (auto &a : args) if (a->op != Op::Constant) return;
      std::vector<double> x, y, out;
      std::uint32_t s = 0;
      auto expand = [&](const Term::Ptr &a, std::vector<double> &v) { a->constant->expandTo(v, vs); };
      switch (t->op) {
        case Op::Add: case Op::Sub: case Op::Mul:
          expand(args[0], x); expand(args[1], y); out.resize(vs);
          for (std::size_t i = 0; i < vs; i++) out[i] = t->op == Op::Add ? x[i] + y[i] : t->op == Op::Sub ? x[i] - y[i] : x[i] * y[i];
          s = std::max(scale[args[0]], scale[args[1]]);
          break;
        case Op::RotateLeftConst: case Op::RotateRightConst: {
          expand(args[0], x); out.resize(vs);
          long long sh = *t->rotation;
          if (t->op == Op::RotateRightConst) sh = -sh;
          sh %= (long long)vs; if (sh < 0) sh += (long long)vs;
          for (std::size_t i = 0; i < vs; i++) out[i] = x[(i + sh) % vs];
          s = scale[args[0]];
        } break;
        case Op::Negate:
          expand(args[0], x); out.resize(vs);
          for (std::size_t i = 0; i < vs; i++) out[i] = -x[i];
          s = scale[args[0]];
          break;
        case Op::Output: case Op::Encode: return;
        case Op::Relinearize: case Op::ModSwitch: case Op::Rescale:
          throw std::logic_error(std::string("Encountered HE specific operation ") + opName(t->op) + " in unencrypted computation");
        default: throw std::logic_error(std::string("Unhandled op ") + opName(t->op));
      }
      auto c = p.makeDenseConstant(out);
      scale[c] = s;
      c->encodeAtScale = s;
      t->replaceAllUsesWith(c);
    });
  }

  // ---- reference eva/common/reduction_balancer.h:28-146 ----
  static void combineReductions(Program &p) {
    traverse(p, true, [&](Term::Ptr &t) {
      if (!t->isInternal() || !(t->op == Op::Add || t->op == Op::Mul)) return;
      auto uses = t->getUses();
      if (uses.size() != 1) return;
      auto &use = uses[0];
      if (use->op != t->op) return;
      while (use->eraseOperand(t))
        for (auto &o : t->getOperands()) use->addOperand(o);
    });
  }
  static void expandReductions(Program &p, Types &type) {
    TermMapOpt<int> scale(p);
    traverse(p, true, [&](Term::Ptr &t) {
      if (t->op == Op::Rescale || t->op == Op::ModSwitch)
        throw std::logic_error("Rescale or ModSwitch encountered, but ReductionLogExpander uses scale as a proxy for level and assumes rescaling has not been performed yet.");
      if (t->numOperands() == 0) scale[t] = (int)t->encodeAtScale.value();
      else if (t->op == Op::Mul) { int s = 0; for (auto &o : t->getOperands()) s += scale.at(o); scale[t] = s; }
      else { int s = 0; for (auto &o : t->getOperands()) s = std::max(s, scale.at(o)); scale[t] = s; }
      if (!(t->op == Op::Add || t->op == Op::Mul) || t->numOperands() <= 2) return;
      // constants / plaintext first, then ciphertexts by scale
      std::map<std::uint32_t, std::vector<Term::Ptr>> sorted;
      for (auto &o : t->getOperands()) {
        std::uint32_t order = 0;
        if (type[o] == Type::Plain || type[o] == Type::Raw) order = 1;
        else if (type[o] == Type::Cipher) order = 2 + (std::uint32_t)scale.at(o);
        sorted[order].push_back(o);
      }
      std::vector<Term::Ptr> ops, next;
      for (auto &e : sorted) ops.insert(ops.end(), e.second.begin(), e.second.end());
      while (ops.size() > 2) {  // pair adjacent operands until two remain
        std::size_t i = 0;
        for (; i + 1 < ops.size(); i += 2) next.push_back(p.makeTerm(t->op, {ops[i], ops[i + 1]}));
        if (i < ops.size()) next.push_back(ops[i]);
        ops.swap(next);
        next.clear();
      }
      t->setOperands(ops);
    });
  }

  // ---- rescaling policies (reference eva/ckks/rescaler.h:27-56 and the four policy headers) ----
  struct RescaleCtx {
    Program &p; Types &type; Scales &scale; std::uint32_t minScale = 0;
    RescaleCtx(Program &p_, Types &t, Scales &s) : p(p_), type(t), scale(s) {
      for (auto &src : p.getSources()) minScale = std::max(minScale, scale[src]);
    }
    Term::Ptr insertRescale(const Term::Ptr &t, std::uint32_t by) {
      auto r = p.makeRescale(t, by);
      type[r] = type[t]; scale[r] = scale[t] - by;
      t->replaceOtherUsesWith(r);
      return r;
    }
    void insertRescaleBetween(const Term::Ptr &a, const Term::Ptr &user, std::uint32_t by) {
      auto r = p.makeRescale(a, by);
      type[r] = type[a]; scale[r] = scale[a] - by;
      user->replaceOperand(a, r);
    }
    void rawScale(const Term::Ptr &t) { std::uint32_t m = 0; for (auto &o : t->getOperands()) m = std::max(m, scale.at(o)); scale[t] = m; }
    // multiply lower-scale operands of an addition by an encoded 1 at the missing scale
    void matchAdditionScales(const Term::Ptr &t, std::uint32_t maxScale) {
      for (auto &o : std::vector<Term::Ptr>(t->getOperands())) {
        if (scale[o] < maxScale && type[o] != Type::Raw) {
          auto one = p.makeUniformConstant(1);
          scale[one] = maxScale - scale[o];
          one->encodeAtScale = scale[one];
          auto mul = p.makeTerm(Op::Mul, {o, one});
          scale[mul] = maxScale;
          t->replaceOperand(o, mul);
        }
      }
    }
  };
  // reference eva/ckks/lazy_waterline_rescaler.h:11-160
  static void rescaleLazyWaterline(Program &p, Types &type, Scales &scale) {
    RescaleCtx c(p, type, scale);
    const std::uint32_t fixed = 60;
    TermMap<bool> pending(p);
    traverse(p, true, [&](Term::Ptr &t) {
      if (t->numOperands() == 0) return;
      if (type[t] == Type::Raw) { c.rawScale(t); return; }
      if (t->op == Op::Rescale) return;
      if (t->op == Op::Mul) {
        std::uint32_t ms = 0;
        for (auto &o : t->getOperands()) ms += scale[o];
        scale[t] = ms;
        if (ms >= fixed + c.minScale) pending[t] = 1; else return;
      } else {
        scale[t] = scale[t->operandAt(0)];
        if (isAddSub(t->op)) {
          std::uint32_t mx = scale[t];
          for (auto &o : t->getOperands()) mx = std::max(mx, scale[o]);
          scale[t] = mx;
          c.matchAdditionScales(t, mx);
        }
        if (!pending[t]) return;
      }
      bool must = false;
      auto uses = t->getUses();
      for (auto &u : uses)
        if (u->op == Op::Mul || u->op == Op::Output || u != uses[0]) { must = true; break; }
      if (must) {
        pending[t] = 0;
        Term::Ptr cur = t;
        std::uint32_t s = scale[cur];
        while (s >= fixed + c.minScale) { cur = c.insertRescale(cur, fixed); s -= fixed; }
      } else {
        for (auto &u : uses) pending[u] = 1;
      }
    });
  }
  // reference eva/ckks/eager_waterline_rescaler.h:11-93
  static void rescaleEagerWaterline(Program &p, Types &type, Scales &scale) {
    RescaleCtx c(p, type, scale);
    const std::uint32_t fixed = 60;
    traverse(p, true, [&](Term::Ptr &t) {
      if (t->numOperands() == 0) return;
      if (type[t] == Type::Raw) { c.rawScale(t); return; }
      if (t->op == Op::Rescale) return;
      if (t->op != Op::Mul) {
        scale[t] = scale[t->operandAt(0)];
        if (isAddSub(t->op)) {
          std::uint32_t mx = scale[t];
          for (auto &o : t->getOperands()) mx = std::max(mx, scale[o]);
          c.matchAdditionScales(t, mx);
          scale[t] = mx;
        }
        return;
      }
      std::uint32_t ms = 0;
      for (auto &o : t->getOperands()) ms += scale[o];
      scale[t] = ms;
      Term::Ptr cur = t;
      while (ms >= fixed + c.minScale) { cur = c.insertRescale(cur, fixed); ms -= fixed; }
    });
  }
  // reference eva/ckks/always_rescaler.h:11-62
  static void rescaleAlways(Program &p, Types &type, Scales &scale) {
    RescaleCtx c(p, type, scale);
    traverse(p, true, [&](Term::Ptr &t) {
      if (t->numOperands() == 0) return;
      if (type[t] == Type::Raw) { c.rawScale(t); return; }
      if (t->op == Op::Rescale) return;
      if (t->op != Op::Mul) { scale[t] = scale[t->operandAt(0)]; return; }
      std::uint32_t ms = 0;
      for (auto &o : t->getOperands()) ms += scale[o];
      scale[t] = ms;
      c.insertRescale(t, ms - c.minScale);
    });
  }
  // reference eva/ckks/minimum_rescaler.h:11-121
  static void rescaleMinimum(Program &p, Types &type, Scales &scale) {
    RescaleCtx c(p, type, scale);
    const std::uint32_t maxRescale = 60;
    traverse(p, true, [&](Term::Ptr &t) {
      if (t->numOperands() == 0) return;
      if (type[t] == Type::Raw) { c.rawScale(t); return; }
      if (t->op == Op::Rescale) return;
      if (t->op != Op::Mul) {
        scale[t] = scale[t->operandAt(0)];
        if (isAddSub(t->op)) {
          std::uint32_t mx = scale[t];
          for (auto &o : t->getOperands()) mx = std::max(mx, scale[o]);
          c.matchAdditionScales(t, mx);
          scale[t] = mx;
        }
        return;
      }
      std::vector<Term::Ptr> ops(t->getOperands());
      std::uint32_t ms = scale[ops[0]] + scale[ops[1]];
      scale[t] = ms;
      std::uint32_t by = std::min(scale[ops[0]], scale[ops[1]]) - c.minScale;
      if (by > maxRescale) by = maxRescale;
      if (2 * by >= maxRescale) {  // rescale both operands before multiplying
        c.insertRescaleBetween(ops[0], t, by);
        if (ops[0] != ops[1]) c.insertRescaleBetween(ops[1], t, by);
        scale[t] = ms - 2 * by;
      } else {
        Term::Ptr cur = t;
        while (ms >= maxRescale + c.minScale) { cur = c.insertRescale(cur, maxRescale); ms -= maxRescale; }
      }
    });
  }

  // ---- reference eva/ckks/encode_inserter.h:11-59 ----
  static void insertEncodes(Program &p, Types &type, Scales &scale) {
    traverse(p, true, [&](Term::Ptr &t) {
      if (t->numOperands() != 2) return;
      auto enc = [&](const Term::Ptr &other, const Term::Ptr &raw) {
        auto e = p.makeTerm(Op::Encode, {raw});
        type[e] = Type::Plain;
        scale[e] = isAddSub(t->op) ? scale[other] : scale[raw];
        e->encodeAtScale = scale[e];
        return e;
      };
      Term::Ptr l = t->operandAt(0), r = t->operandAt(1);
      if (type[l] == Type::Cipher && type[r] == Type::Raw) t->replaceOperand(r, enc(l, r));
      l = t->operandAt(0); r = t->operandAt(1);
      if (type[r] == Type::Cipher && type[l] == Type::Raw) t->replaceOperand(l, enc(r, l));
    });
  }

  // ---- reference eva/ckks/lazy_relinearizer.h:11-94 / eager_relinearizer.h:11-54 ----
  static void relinearize(Program &p, Types &type, Scales &scale, bool lazy) {
    auto encMul = [&](const Term::Ptr &t) {
      if (t->op != Op::Mul) return false;
      for (auto &o : t->getOperands()) if (type[o] != Type::Cipher) return false;
      return true;
    };
    auto insert = [&](const Term::Ptr &t) {
      auto r = p.makeTerm(Op::Relinearize, {t});
      type[r] = type[t]; scale[r] = scale[t];
      t->replaceOtherUsesWith(r);
    };
    if (!lazy) {
      traverse(p, true, [&](Term::Ptr &t) { if (t->numOperands() && encMul(t)) insert(t); });
      return;
    }
    TermMap<bool> pending(p);
    traverse(p, true, [&](Term::Ptr &t) {
      if (t->numOperands() == 0) return;
      if (encMul(t)) pending[t] = 1;
      else if (!pending[t]) return;
      bool must = false;
      auto uses = t->getUses();
      for (auto &u : uses)
        if (encMul(u) || isRot(u->op) || u->op == Op::Output || u != uses[0]) { must = true; break; }
      if (must) insert(t);
      else for (auto &u : uses) pending[u] = 1;
    });
  }

  // ---- reference eva/ckks/mod_switcher.h:11-95 (backward pass + finalisation) ----
  static void switchModuli(Program &p, Types &type, Scales &scale) {
    TermMap<std::uint32_t> level(p);  // reverse level: sinks 0
    std::vector<Term::Ptr> encodes;
    traverse(p, false, [&](Term::Ptr &t) {
      if (t->numUses() == 0) return;
      if (type[t] == Type::Raw) return;
      if (t->op == Op::Encode) encodes.push_back(t);
      std::map<std::uint32_t, std::vector<Term::Ptr>> useLevels;
      for (auto &u : t->getUses()) useLevels[level[u]].push_back(u);
      std::uint32_t tl = 0;
      if (useLevels.size() > 1) {
        auto it = useLevels.rbegin();
        tl = it->first;
        ++it;
        Term::Ptr cur = t;
        std::uint32_t curLevel = tl;
        for (; it != useLevels.rend(); ++it) {
          while (curLevel > it->first) {
            auto ms = p.makeTerm(Op::ModSwitch, {cur});
            scale[ms] = scale[cur];
            level[ms] = curLevel;
            cur = ms;
            --curLevel;
          }
          for (auto &u : it->second) u->replaceOperand(t, cur);
        }
      } else tl = useLevels.begin()->first;
      if (t->op == Op::Rescale) ++tl;
      level[t] = tl;
    });
    auto sources = p.getSources();
    std::uint32_t maxLevel = 0;
    for (auto &s : sources) maxLevel = std::max(maxLevel, level[s]);
    for (auto &s : sources) s->encodeAtLevel = maxLevel - level[s];
    for (auto &e : encodes) e->encodeAtLevel = maxLevel - level[e];
  }

  // ---- reference eva/ckks/seal_lowering.h:11-30: plain - cipher  =>  plain + (-cipher) ----
  static void lowerPlainMinusCipher(Program &p, Types &type) {
    traverse(p, true, [&](Term::Ptr &t) {
      if (t->op == Op::Sub && type[t->operandAt(0)] != Type::Cipher && type[t->operandAt(1)] == Type::Cipher) {
        auto neg = p.makeTerm(Op::Negate, {t->operandAt(1)});
        auto add = p.makeTerm(Op::Add, {t->operandAt(0), neg});
        t->replaceAllUsesWith(add);
      }
    });
  }

  void transform(Program &p, Types &types, Scales &scales) {
    deduceTypes(p, types);
    foldConstants(p, scales);
    if (config_.balanceReductions) { combineReductions(p); expandReductions(p, types); }
    switch (config_.rescaler) {
      case Rescaler::Minimum: rescaleMinimum(p, types, scales); break;
      case Rescaler::Always: rescaleAlways(p, types, scales); break;
      case Rescaler::EagerWaterline: rescaleEagerWaterline(p, types, scales); break;
      case Rescaler::LazyWaterline: rescaleLazyWaterline(p, types, scales); break;
    }
    deduceTypes(p, types);
    insertEncodes(p, types, scales);
    deduceTypes(p, types);
    relinearize(p, types, scales, config_.lazyRelinearize);
    deduceTypes(p, types);
    switchModuli(p, types, scales);
    deduceTypes(p, types);
    lowerPlainMinusCipher(p, types);
  }

  // ---- validation (reference levels_checker.h, parameter_checker.h, scales_checker.h) ----
  void validate(Program &p, Types &types, Scales &) {
    TermMap<std::size_t> levels(p);
    traverse(p, true, [&](Term::Ptr &t) {
      if (t->numOperands() == 0) { levels[t] = t->encodeAtLevel.value_or(0); return; }
      bool have = false; std::size_t lv = 0;
      for (auto &o : t->getOperands())
        if (types[o] == Type::Cipher) {
          if (!have) { lv = levels[o]; have = true; }
          else if (levels[o] != lv) throw std::logic_error("Compiled program has operands at different levels");
        }
      if (t->op == Op::Rescale || t->op == Op::ModSwitch) ++lv;
      levels[t] = lv;
    });
    TermMap<std::vector<std::uint32_t>> parms(p);
    try {
      traverse(p, true, [&](Term::Ptr &t) {
        if (types[t] == Type::Raw || t->op == Op::Encode) return;
        auto &mine = parms[t];
        if (t->numOperands() == 0) { mine.assign(t->encodeAtLevel.value_or(0), 0); return; }
        for (auto &o : t->getOperands()) {
          auto &op = parms[o];
          if (op.empty()) continue;
          if (mine.empty()) { mine = op; continue; }
          if (op.size() != mine.size()) throw Inconsistent("Two operands require different number of primes");
          for (std::size_t i = 0; i < mine.size(); i++) {
            if (mine[i] == 0) mine[i] = op[i];
            else if (op[i] != 0 && op[i] != mine[i]) throw Inconsistent("Primes required by two operands do not match");
          }
        }
        if (t->op == Op::ModSwitch) mine.push_back(0);
        else if (t->op == Op::Rescale) mine.push_back(t->rescaleDivisor.value());
      });
    } catch (const Inconsistent &) {
      switch (config_.rescaler) {
        case Rescaler::Minimum: throw std::runtime_error("The 'minimum' rescaler produced inconsistent parameters. Note that this rescaling policy is not general and thus will not work for all programs. Please use a different rescaler for this program.");
        case Rescaler::Always: throw std::runtime_error("The 'always' rescaler produced inconsistent parameters. Note that this rescaling policy is not general. It is only guaranteed to work for programs that have equal scale for all inputs and constants.");
        default: throw std::runtime_error("The current rescaler produced inconsistent parameters. This is a bug, as this rescaler should be able to handle all programs.");
      }
    }
    TermMapOpt<std::uint32_t> sc(p);
    traverse(p, true, [&](Term::Ptr &t) {
      if (types[t] == Type::Raw) return;
      auto zero = [] { throw std::logic_error("Compiled program results in a 0 scale term"); };
      if (t->op == Op::Input || t->op == Op::Encode) {
        sc[t] = t->encodeAtScale.value();
        if (sc.at(t) == 0) { if (t->op == Op::Input) throw std::runtime_error("Program has an input with 0 scale"); zero(); }
      } else if (t->op == Op::Mul) {
        std::uint32_t s = 0;
        for (auto &o : t->getOperands()) s += sc.at(o);
        if (!s) zero();
        sc[t] = s;
      } else if (t->op == Op::Rescale) {
        std::uint32_t s = sc.at(t->operandAt(0)) - t->rescaleDivisor.value();
        if (!s) zero();
        sc[t] = s;
      } else if (isAddSub(t->op)) {
        std::uint32_t s = 0;
        for (auto &o : t->getOperands()) {
          if (!s) s = sc.at(o);
          else if (s != sc.at(o)) throw std::logic_error("Addition or subtraction in program has operands of non-equal scale");
        }
        if (!s) zero();
        sc[t] = s;
      } else {
        std::uint32_t s = sc.at(t->operandAt(0));
        if (!s) zero();
        sc[t] = s;
      }
    });
  }
  struct Inconsistent : std::runtime_error { explicit Inconsistent(const std::string &m) : std::runtime_error(m) {} };

  // ---- reference encryption_parameter_selector.h:15-199, rotation_keys_selector.h:16-54,
  //      ckks_compiler.h:136-253 ----
  CKKSParameters selectParameters(Program &p, Types &types, Scales &scales) {
    TermMap<std::vector<std::uint32_t>> chain(p);
    std::set<int> rotations;
    traverse(p, true, [&](Term::Ptr &t) {
      if (isRot(t->op) && types[t] != Type::Raw) rotations.insert(t->op == Op::RotateRightConst ? -*t->rotation : *t->rotation);
      if (types[t] == Type::Raw || t->op == Op::Encode || t->numOperands() == 0) return;
      auto &mine = chain[t];
      for (auto &o : t->getOperands()) if (chain[o].size() > mine.size()) mine = chain[o];
      if (t->op == Op::Rescale) mine.push_back(t->rescaleDivisor.value());
    });
    std::vector<std::uint32_t> parms;
    std::uint32_t maxOut = 0, maxParm = 0;
    std::size_t maxLen = 0;
    for (auto &e : p.getOutputs()) {
      auto &o = e.second;
      maxOut = std::max(maxOut, o->range.value() + scales[o]);
      maxLen = std::max(maxLen, chain[o].size());
      for (auto v : chain[o]) maxParm = std::max(maxParm, v);
    }
    if (maxOut > 60) {
      maxParm = 60;
      while (maxOut >= 60) { parms.push_back(60); maxOut -= 60; }
      if (maxOut > 0) parms.push_back(std::max(20u, maxOut));
    } else {
      maxParm = std::max(maxParm, maxOut);
      parms.push_back(maxParm);
    }
    for (auto &e : p.getOutputs())
      if (chain[e.second].size() == maxLen) { parms.insert(parms.end(), chain[e.second].rbegin(), chain[e.second].rend()); break; }
    parms.push_back(maxParm);  // the key-switching prime

    CKKSParameters out;
    out.primeBits = parms;
    out.rotations = rotations;
    int bitCount = 0;
    for (auto b : parms) bitCount += (int)b;
    if (config_.securityLevel > 256)
      throw std::runtime_error("EVA has support for up to 256 bit security, but " + std::to_string(config_.securityLevel) + " bit security was requested.");
    std::size_t degree = 1024;
    int maxSeen = 0;
    for (;;) {
      int mb = heStdMaxBits(config_.securityLevel, config_.quantumSafe, degree);
      maxSeen = std::max(maxSeen, mb);
      if (mb == 0) throw std::runtime_error("Program requires a " + std::to_string(bitCount) + " bit modulus, but parameters are available for a maximum of " + std::to_string(maxSeen));
      if (mb >= bitCount) break;
      degree *= 2;
    }
    out.polyModulusDegree = (std::uint32_t)degree;
    const std::uint32_t slots = out.polyModulusDegree / 2;
    if (config_.warnVecSize && slots > p.getVecSize())
      warn("Program specifies vector size %i while at least %i slots are required for security. This does not affect correctness, as the smaller vector size will be transparently emulated. However, using a vector size up to %i would come at no additional cost.", (int)p.getVecSize(), (int)slots, (int)slots);
    if (slots < p.getVecSize()) {
      if (config_.warnVecSize)
        warn("Program uses vector size %i while only %i slots are required for security. This does not affect correctness, but higher performance may be available with a smaller vector size.", (int)p.getVecSize(), (int)slots);
      out.polyModulusDegree = 2 * p.getVecSize();
    }
    if (verbosity() >= 1) {
      std::printf("EVA: Encryption parameters for %s are:\n  Q = [", p.getName().c_str());
      for (std::size_t i = 0; i < parms.size(); i++) std::printf("%s%u", i ? "," : "", parms[i]);
      std::printf("] (total bits %i)\n  N = %u (available slots %u)\n  Rotation keys: %zu\n", bitCount, out.polyModulusDegree, out.polyModulusDegree / 2, rotations.size());
    }
    return out;
  }

  CKKSConfig config_;
};

// ---- slot packing: k instances of a compiled program whose vec_size v is below N/2, in every ciphertext ----
// Instance b's slot i sits at packed slot i*k + b, which fills k*v slots.  A rotation by r*k of the packed vector (period v*k) is
// the rotation by r of every instance: (i*k + b + r*k) mod (v*k) = ((i + r) mod v)*k + b.  Every other op acts slot by slot.  So the
// packed program is the same program with vec_size v*k, every rotation step r replaced by (r mod v)*k, and every constant of m values
// replaced by its m*k interleaved values c'[i*k + b] = c[i] (a uniform constant keeps its one value).  Types, scales, levels, rescales,
// relinearizations, mod-switches and the input and output names stay.  The parameters keep prime_bits and N, with the packed
// program's rotation steps; the signature keeps its inputs' encodings with vec_size v*k.  What runs it (planner, executor, keys)
// sees an ordinary program with the same terms.  k = 1 returns copies of the input.
inline std::tuple<std::unique_ptr<Program>, CKKSParameters, CKKSSignature> packProgram(const Program &prog, const CKKSParameters &params,
                                                                                       const CKKSSignature &sig, int k) {
  const std::size_t v = prog.getVecSize(), slots = params.polyModulusDegree / 2;
  if (k < 1 || (k & (k - 1))) throw std::invalid_argument("pack_program: k = " + std::to_string(k) + " is not a power of two");
  if ((std::size_t)sig.vecSize != v)
    throw std::invalid_argument("pack_program: the signature's vec_size " + std::to_string(sig.vecSize) + " differs from the program's vec_size " + std::to_string(v));
  if ((std::size_t)k * v > slots)
    throw std::invalid_argument("pack_program: k = " + std::to_string(k) + " instances of vec_size " + std::to_string(v) + " need " + std::to_string(k * v) +
                                " slots, more than the " + std::to_string(slots) + " of N = " + std::to_string(params.polyModulusDegree));
  if (k == 1) return std::make_tuple(prog.deepCopy(), params, sig);
  auto packed = std::make_unique<Program>(prog.getName() + ".pack" + std::to_string(k), v * k);
  std::map<const Term *, std::string> inName, outName;
  for (auto &e : prog.getInputs()) inName[e.second.get()] = e.first;
  for (auto &e : prog.getOutputs()) outName[e.second.get()] = e.first;
  std::map<std::uint64_t, Term::Ptr> copy;
  std::map<std::uint64_t, Type> type;   // the compiler's type deduction: rotation keys are selected for non-Raw rotations only
  std::set<int> rotations;
  for (auto &t : prog.toposort()) {
    std::vector<Term::Ptr> ops;
    Type ty = Type::Raw;
    for (auto &o : t->getOperands()) {
      ops.push_back(copy.at(o->index));
      if (type.at(o->index) == Type::Cipher) ty = Type::Cipher;
    }
    if (t->op == Op::Encode) ty = Type::Plain;
    else if (t->op == Op::Input) ty = t->type.value();
    type[t->index] = ty;
    Term::Ptr n = t->op == Op::Input ? packed->makeInput(inName.at(t.get()), ty)
                : t->op == Op::Output ? packed->makeOutput(outName.at(t.get()), ops.at(0))
                : packed->makeTerm(t->op, ops);
    n->copyAttributesFrom(*t);
    if (t->op == Op::RotateLeftConst || t->op == Op::RotateRightConst) {
      const long long r = ((long long)*t->rotation % (long long)v + (long long)v) % (long long)v;
      n->rotation = (std::int32_t)(r * k);
      if (ty != Type::Raw) rotations.insert(t->op == Op::RotateLeftConst ? *n->rotation : -*n->rotation);
    }
    if (t->constant) {
      const std::vector<double> &c = t->constant->values();
      std::vector<double> interleaved;
      if (c.size() == 1) interleaved = c;
      else {
        interleaved.reserve(c.size() * k);
        for (double x : c) interleaved.insert(interleaved.end(), (std::size_t)k, x);
      }
      n->constant = std::make_shared<ConstantValue>(t->constant->size() * k, std::move(interleaved));
    }
    copy[t->index] = n;
  }
  CKKSParameters pp = params;
  pp.rotations = rotations;
  return std::make_tuple(std::move(packed), std::move(pp), CKKSSignature((int)(v * k), sig.inputs));
}

}  // namespace evab
