// pymodule.cpp -- pybind11 module `eva_b200._eva_b200`: the Python-facing
// surface of the backend, name-compatible with the reference's `_eva` module
// (python/eva/wrapper.cpp:26-246) for Program/Term/Op/Type/evaluate/
// CKKSParameters/CKKSSignature/CKKSEncodingInfo/generate_keys/*Valuation/
// *Public.encrypt/execute/*Secret.decrypt, plus a few test/benchmark hooks
// (raw key/ciphertext injection, device-resident execution).
#include "backend.hpp"
#include "compiler.hpp"
#include "reference_eval.hpp"
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>
#include <optional>

namespace py = pybind11;
using namespace evab;
typedef py::array_t<std::uint64_t, py::array::c_style | py::array::forcecast> u64arr;

static std::vector<u64> toVec(const u64arr &a) { return std::vector<u64>(a.data(), a.data() + a.size()); }
static HostBuf toHostBuf(const u64arr &a) { HostBuf b(a.size()); std::memcpy(b.data(), a.data(), a.size() * 8); return b; }

// key material loaded from files / callers: shapes are checked against (k, N) before anything reaches the device
static void requireShape(const u64arr &a, std::initializer_list<std::size_t> shape, const char *what) {
  bool ok = (std::size_t)a.ndim() == shape.size();
  std::size_t i = 0;
  for (std::size_t d : shape) { if (ok && (std::size_t)a.shape(i) != d) ok = false; i++; }
  if (!ok) throw std::runtime_error(std::string(what) + " does not match the parameters (modulus count / degree)");
}

// a key seed from Python bytes: exactly 32 of them
static KeySeed toSeed(const py::bytes &b, const char *what) {
  const std::string v = b;
  if (v.size() != 32) throw std::invalid_argument(std::string(what) + " seed must be exactly 32 bytes (got " + std::to_string(v.size()) + ")");
  KeySeed s;
  std::memcpy(s.data(), v.data(), 32);
  return s;
}
static py::bytes fromSeed(const KeySeed &s) { return py::bytes(reinterpret_cast<const char *>(s.data()), 32); }

// test hook of B200Public / B200Secret: Encryptor::encrypt_symmetric of a plaintext polynomial [ell][N] with an EXPLICIT seed and
// error -> the full ciphertext [2][ell][N] (c1: the seed's expansion)
static u64arr encryptSeededPoly(const std::shared_ptr<Shared> &s, const u64arr &pt, const py::bytes &seed, const std::vector<int> &e) {
  if (pt.ndim() != 2 || (std::size_t)pt.shape(1) != s->dev->N()) throw std::runtime_error("plaintext array must be [ell][N]");
  const KeySeed sd = toSeed(seed, "ciphertext");
  const int ell = (int)pt.shape(0);
  DBuf d(s->dev, pt.size());
  s->dev->upload(d.get(), pt.data(), pt.size() * 8);
  DBuf ct = s->client->encryptSeededWith(s->keys, d.get(), ell, sd, e);
  u64arr a({(std::size_t)2, (std::size_t)ell, (std::size_t)s->dev->N()});
  s->dev->download(a.mutable_data(), ct.get(), a.size() * 8);
  s->dev->sync();
  return a;
}

// set_options: one argument list for B200Public and for the planner test hook (_plan), which parses its options dict through it
static ExecOptions &optionsOf(B200Public &p) { return p.options; }
static ExecOptions &optionsOf(B200Server &s) { return s.pub().options; }
static ExecOptions &optionsOf(ExecOptions &o) { return o; }
// compact_outputs belongs to the context, not to its plans (the planner hook has none)
static int *compactOf(B200Public &p) { return &p.compactOutputs; }
static int *compactOf(B200Server &s) { return &s.pub().compactOutputs; }
static int *compactOf(ExecOptions &) { return nullptr; }
template <class Self>
static void setOptions(Self &self, int streams, bool graph, bool cache, bool dedup, int fuse, bool fuseSums, bool hoist, bool uniformEncode, bool dedupTerms,
                       bool hoistModUp, bool approxHoist, int rotationChunk, std::size_t arenaLimit, bool rotationSums, int compactOutputs) {
  if (compactOutputs < 0 || compactOutputs > 52)
    throw py::value_error("compact_outputs (" + std::to_string(compactOutputs) + ") must be 0 (off) or the precision in bits, 1 .. 52");
  if (int *c = compactOf(self)) *c = compactOutputs;
  ExecOptions &o = optionsOf(self);
  o.numStreams = streams; o.useGraph = graph; o.cacheConstants = cache; o.dedupConstants = dedup;
  o.fuse = fuse; o.fuseSums = fuseSums; o.hoistRotations = hoist; o.uniformEncode = uniformEncode;
  o.dedupTerms = dedupTerms; o.hoistModUp = hoistModUp; o.approxHoist = approxHoist; o.rotationChunk = rotationChunk;
  o.arenaLimit = arenaLimit; o.rotationSums = rotationSums;
}
template <class Class>
static void defSetOptions(Class &cls) {
  cls.def("set_options", &setOptions<typename Class::type>,
          py::arg("num_streams") = 8, py::arg("use_graph") = true, py::arg("cache_constants") = true, py::arg("dedup_constants") = true,
          py::arg("fuse") = 1, py::arg("fuse_sums") = true, py::arg("hoist_rotations") = true, py::arg("uniform_encode") = true, py::arg("dedup_terms") = true, py::arg("hoist_mod_up") = true, py::arg("approx_hoist") = false, py::arg("rotation_chunk") = 16,
          py::arg("arena_limit") = 0, py::arg("rotation_sums") = true, py::arg("compact_outputs") = 0,
          "arena_limit: bytes one plan's arena may take (0: the free device memory when the plan is built).  A plan whose one-offset-per-value "
          "layout does not fit reuses the storage of dead values; if even that exceeds the limit, building the plan raises RuntimeError.  "
          "rotation_sums: sums of rotations of one ciphertext weighted by scalar constants run as one bit-exact evab_rotate_wsum call (approx_hoist takes precedence).  "
          "compact_outputs: 0 (off) or p in 1 .. 52: every size-2 output ciphertext is switched on the GPU to the modulus 2^b its declared range "
          "and p bits after the binary point need, and returned bit-packed (B200Valuation kind \"compact_cipher\"); builds no plan");
}

// execute_batch_async handle: the batch plus the Python objects it reads from.  Destroyed with the GIL held (the batch first:
// it waits for its copies before the valuations may go)
struct PyPending {
  std::shared_ptr<evab::PendingBatch> batch;
  py::object program, inputs;
  ~PyPending() { batch.reset(); }
};

// test hook shared by B200Public and B200Server: the value of a term in instance b of a plan's arena
static py::object debugValue(B200Public &p, Program &prog, std::uint64_t index, int batch, int b) {
  Executor &ex = p.executorFor(prog, batch);
  const ValueInfo &vi = ex.info(index);
  auto dev = p.shared()->dev;
  if (vi.kind == Kind::Raw) return py::cast(ex.rawValue(index, b));
  if (vi.kind == Kind::None || vi.fused) return py::none();   // fused away: never materialised
  if (!ex.intact(index))
    throw std::runtime_error("term " + std::to_string(index) + " is not kept by this plan's packed arena (its storage is reused after its last "
                             "use); only inputs, outputs and cached constants can be read back");
  const std::size_t polys = vi.kind == Kind::Cipher ? vi.size : 1;
  u64arr a({polys, (std::size_t)vi.ell, (std::size_t)dev->N()});
  dev->sync();
  dev->download(a.mutable_data(), ex.valuePtr(index, b), a.size() * 8);
  dev->sync();
  return py::make_tuple(a, vi.scale);
}

PYBIND11_MODULE(_eva_b200, m) {
  m.doc() = "H100-native (sm_90a) EVA backend";

  py::enum_<Op>(m, "Op")
      .value("Undef", Op::Undef).value("Input", Op::Input).value("Output", Op::Output).value("Constant", Op::Constant)
      .value("Negate", Op::Negate).value("Add", Op::Add).value("Sub", Op::Sub).value("Mul", Op::Mul)
      .value("RotateLeftConst", Op::RotateLeftConst).value("RotateRightConst", Op::RotateRightConst)
      .value("Relinearize", Op::Relinearize).value("ModSwitch", Op::ModSwitch).value("Rescale", Op::Rescale).value("Encode", Op::Encode);
  py::enum_<Type>(m, "Type").value("Undef", Type::Undef).value("Cipher", Type::Cipher).value("Raw", Type::Raw).value("Plain", Type::Plain);

  py::class_<Term, std::shared_ptr<Term>>(m, "Term", "EVA's native Term class")
      .def_readonly("op", &Term::op, "The operation performed by this term")
      .def_readonly("index", &Term::index)
      .def_property_readonly("operands", &Term::getOperands)
      .def_property_readonly("attributes", [](const Term &t) {
        py::dict d;
        if (t.rescaleDivisor) d["RescaleDivisorAttribute"] = *t.rescaleDivisor;
        if (t.rotation) d["RotationAttribute"] = *t.rotation;
        if (t.type) d["TypeAttribute"] = *t.type;
        if (t.range) d["RangeAttribute"] = *t.range;
        if (t.encodeAtScale) d["EncodeAtScaleAttribute"] = *t.encodeAtScale;
        if (t.encodeAtLevel) d["EncodeAtLevelAttribute"] = *t.encodeAtLevel;
        if (t.constant) d["ConstantValueAttribute"] = t.constant->values();
        return d;
      })
      .def("_set_attributes", [](Term &t, const py::dict &d) {  // fixture loading / tests
        for (auto item : d) {
          const std::string k = py::cast<std::string>(item.first);
          if (k == "RescaleDivisorAttribute") t.rescaleDivisor = py::cast<std::uint32_t>(item.second);
          else if (k == "RotationAttribute") t.rotation = py::cast<std::int32_t>(item.second);
          else if (k == "TypeAttribute") t.type = py::cast<Type>(item.second);
          else if (k == "RangeAttribute") t.range = py::cast<std::uint32_t>(item.second);
          else if (k == "EncodeAtScaleAttribute") t.encodeAtScale = py::cast<std::uint32_t>(item.second);
          else if (k == "EncodeAtLevelAttribute") t.encodeAtLevel = py::cast<std::uint32_t>(item.second);
          else throw std::runtime_error("unknown attribute " + k);
        }
      });

  py::class_<Program>(m, "Program", "EVA's native Program class")
      .def(py::init<std::string, std::uint64_t>(), py::arg("name"), py::arg("vec_size"))
      .def_property("name", &Program::getName, &Program::setName, "The name of this program")
      .def_property_readonly("vec_size", &Program::getVecSize, "The number of elements for all vectors in this program")
      .def_property_readonly("inputs", &Program::getInputs, "A dictionary from input names to terms")
      .def_property_readonly("outputs", &Program::getOutputs, "A dictionary from output names to terms")
      .def("set_output_ranges", [](const Program &p, std::uint32_t range) { for (auto &e : p.getOutputs()) e.second->range = range; }, py::arg("range"))
      .def("set_input_scales", [](const Program &p, std::uint32_t scale) { for (auto &s : p.getSources()) s->encodeAtScale = scale; }, py::arg("scale"))
      .def("to_DOT", &Program::toDOT)
      .def("terms", &Program::toposort, "All live terms in topological order")
      .def("_make_term", &Program::makeTerm, py::keep_alive<0, 1>())
      .def("_make_left_rotation", &Program::makeLeftRotation, py::keep_alive<0, 1>())
      .def("_make_right_rotation", &Program::makeRightRotation, py::keep_alive<0, 1>())
      .def("_make_dense_constant", &Program::makeDenseConstant, py::keep_alive<0, 1>())
      .def("_make_uniform_constant", &Program::makeUniformConstant, py::keep_alive<0, 1>())
      .def("_make_input", &Program::makeInput, py::keep_alive<0, 1>())
      .def("_make_output", &Program::makeOutput, py::keep_alive<0, 1>());

  m.def("evaluate", &evaluate, py::arg("program"), py::arg("inputs"), "Evaluate the program without homomorphic encryption");
  // test hook: the arena packer alone (host/arena_packer.hpp).  steps: [(stream, [earlier steps waited on])];
  // buffers: [(words, writer step, [reader steps], pinned)] -> (offsets, added waits [(step, earlier step)], peak words)
  m.def("_pack_arena", [](const std::vector<std::tuple<int, std::vector<int>>> &steps,
                          const std::vector<std::tuple<std::size_t, int, std::vector<int>, bool>> &buffers) {
    std::vector<PackStep> ps;
    for (auto &s : steps) ps.push_back(PackStep{std::get<0>(s), std::get<1>(s)});
    std::vector<PackBuffer> pb;
    for (auto &b : buffers) pb.push_back(PackBuffer{std::get<0>(b), std::get<1>(b), std::get<2>(b), std::get<3>(b)});
    PackResult r = packArena(ps, pb);
    return py::make_tuple(r.offsets, r.waits, r.peak);
  }, py::arg("steps"), py::arg("buffers"));
  // test hooks: a residency policy alone (host/slot_cache.hpp).  Replay batches of tenant ids through a cache of `regions` regions;
  // an entry ("remove", t) drops tenant t instead.  Return (per entry: the region of every instance (-1: draws) and [(tenant,
  // region, evicted or -1)] -- _c1_cache adds the tenants holding a region --, the error message, or None for a removal; fills;
  // evictions).  _slot_cache: the key pager's (assignAll); _c1_cache: the c1 store's (assignByCount)
  auto replayRegionCache = [](int regions, const std::vector<py::object> &ops, bool keySlots) {
    RegionCache c(regions);
    py::list results;
    for (auto &op : ops) {
      if (py::isinstance<py::tuple>(op)) {   // ("remove", tenant)
        c.drop(py::cast<int>(op.cast<py::tuple>()[1]));
        results.append(py::none());
        continue;
      }
      std::vector<RegionCache::Fill> fills;
      try {
        const std::vector<int> batch = op.cast<std::vector<int>>();
        std::vector<int> r = keySlots ? c.assignAll(batch, fills) : c.assignByCount(batch, fills);
        py::list fl;
        for (auto &f : fills) fl.append(py::make_tuple(f.tenant, f.region, f.evicted));
        if (keySlots) results.append(py::make_tuple(r, fl));
        else results.append(py::make_tuple(r, fl, c.holders()));
      } catch (const std::invalid_argument &e) {
        results.append(py::str(e.what()));
      }
    }
    return py::make_tuple(results, c.fills(), c.evictions());
  };
  m.def("_slot_cache", [=](int slots, const std::vector<py::object> &ops) { return replayRegionCache(slots, ops, true); },
        py::arg("slots"), py::arg("batches"));
  m.def("_c1_cache", [=](int regions, const std::vector<py::object> &ops) { return replayRegionCache(regions, ops, false); },
        py::arg("regions"), py::arg("batches"));
  // test hook: the ciphertext store's layout (CipherStore) without a device: (store_entry_bytes for k primes at degree N, the host
  // bytes of a paged entry at ell residues, seeded: stored from a seeded ciphertext)
  m.def("_store_bytes", [](int k, u64 N, const std::string &storeStorage, int ell, bool seeded) {
    return py::make_tuple(CipherStore::entryWords(k, N, CipherStore::seededLayout(storeStorage)) * 8, CipherStore::hostWords(ell, N, seeded) * 8);
  }, py::arg("k"), py::arg("N"), py::arg("store_storage"), py::arg("ell"), py::arg("seeded"));
  // test hook: the planner alone (host/planner.hpp), without a device.  options: set_options' keywords; arena_limit 0 is no limit
  // here.  The scratch sizes are stand-ins derived from N and ell (the layout's invariants hold for any sizes)
  py::class_<ExecOptions> planOptions(m, "_PlanOptions");
  planOptions.def(py::init<>());
  defSetOptions(planOptions);
  // galois_elements: the elements that have keys (None: every step has its own).  Besides the plan's shape it returns "chains" (every
  // key-switched rotation of the program -> the steps it applies, composeRotations), "sources" (hops and composed rotations -> the
  // term each reads) and "rotations" (every rotation the plan issues: (term, the term it reads, step))
  m.def("_plan", [](Program &prog, std::uint64_t N, int k, const py::dict &options, int batch, std::optional<std::set<u64>> galoisElements) {
    py::object holder = py::cast(ExecOptions{});
    holder.attr("set_options")(**options);
    ExecOptions opt = holder.cast<ExecOptions>();
    opt.batch = batch;
    WorkSizes ws;
    ws.keyswitch = ws.rotateModupExt = [N](int ell) { return (std::size_t)(ell + 1) * ell * N * 8; };
    ws.rescale = [N](int size) { return (std::size_t)size * N * 8; };
    ws.rotateModupMany = [N](int ell, int n) { return (std::size_t)n * (ell + 1) * N * 8; };
    ws.rotateWsum = [N](int ell, int n, int nout) { return (std::size_t)(n + nout) * (ell + 1) * N * 8; };
    ws.lazyRotsum = [N](int ell, int nout) { return (std::size_t)nout * (ell + 1) * N * 8; };
    ws.encode = [N](int count) { return (std::size_t)count * N * 16; };
    const Plan p = buildPlan(prog, opt, N, k, opt.arenaLimit ? opt.arenaLimit : SIZE_MAX, ws, galoisElements ? &*galoisElements : nullptr);
    static const char *kinds[] = {"Term", "Hoist", "RotationChunk", "RotationSum"};
    py::list steps, regions;
    for (auto &st : p.steps) steps.append(py::make_tuple(kinds[(int)st.kind], st.term->index, st.stream, st.waits, st.record));
    for (auto &r : p.regions) regions.append(py::make_tuple(p.laidWords(r), r.off, r.writer, r.readers, r.pinned));
    py::dict values;   // materialised values: (offset, words, region)
    for (auto &t : p.order)
      if (int r = p.storage[t->index]; r >= 0) {
        const ValueInfo &v = p.vals[t->index];
        const std::size_t rows = v.kind == Kind::Cipher ? (std::size_t)v.size * v.ell : v.ell + (t->op == Op::Encode && p.groups[p.groupIndex.at(t->index)].withP);
        values[py::int_(t->index)] = py::make_tuple(v.off, rows * N, r);
      }
    py::dict d, sources;
    py::list rotations;
    for (auto &kv : p.chainSrc) sources[py::int_(kv.first)] = kv.second->index;
    p.forEachRotation([&](const Term *r, bool) { rotations.append(py::make_tuple(r->index, p.src(r)->index, p.stepOf(r))); });
    d["steps"] = steps; d["regions"] = regions; d["values"] = values; d["stride"] = p.stride; d["stats"] = p.planStats();
    d["chains"] = p.chain; d["sources"] = sources; d["rotations"] = rotations;
    return d;
  }, py::arg("program"), py::arg("N"), py::arg("k"), py::arg("options") = py::dict(), py::arg("batch") = 1, py::arg("galois_elements") = py::none());
  // test hook: the steps that get a Galois key under generate_keys / B200Server(rotation_keys=...)
  m.def("_rotation_key_steps", &rotationKeySteps, py::arg("params"), py::arg("rotation_keys"));
  // test hook: the width rule of compact responses (backend.hpp compactShape) -> (compact, shift, bits, compact scale)
  // range None: the output declares none; cipher / size: the output's kind and polynomial count
  m.def("_compact_shape", [](const std::vector<u64> &primes, int ell, double scale, std::optional<std::uint32_t> range, int precision, u64 N, int size,
                             bool cipher) {
    if (ell < 1 || ell > (int)primes.size()) throw std::invalid_argument("ell out of range");
    const CompactShape c = compactShape(primes, cipher, size, ell, scale, range, precision, N);
    return py::make_tuple(c.compact, c.shift, c.bits, c.scale);
  }, py::arg("primes"), py::arg("ell"), py::arg("scale"), py::arg("range"), py::arg("precision"), py::arg("N"), py::arg("size") = 2,
     py::arg("cipher") = true);
  m.def("set_num_threads", [](int) {}, py::arg("num_threads"),
        "Kept for API compatibility: the DAG is scheduled on CUDA streams, not CPU threads.");
  py::class_<int>(m, "_GaloisGuard").def(py::init());

  py::module mckks = m.def_submodule("_ckks", "CKKS compiler types");
  py::class_<CKKSCompiler>(mckks, "CKKSCompiler")
      .def(py::init(), "Create a compiler with the default config")
      .def(py::init<std::unordered_map<std::string, std::string>>(), py::arg("config"), "Create a compiler with a custom config (dict from strings to strings)")
      .def("compile", &CKKSCompiler::compile, py::arg("program"),
           "Compile a program for CKKS; returns (compiled Program, CKKSParameters, CKKSSignature)");
  mckks.def("pack_program", &packProgram, py::arg("program"), py::arg("params"), py::arg("signature"), py::arg("k"),
            "k instances of a compiled program in every ciphertext: returns (packed Program, CKKSParameters, CKKSSignature) with "
            "vec_size k * vec_size; instance b's slot i is packed slot i * k + b (the inputs are left untouched)");
  py::class_<CKKSParameters>(mckks, "CKKSParameters", "Abstract encryption parameters for CKKS")
      .def(py::init([](std::vector<std::uint32_t> bits, std::set<int> rots, std::uint32_t n) { CKKSParameters p; p.primeBits = bits; p.rotations = rots; p.polyModulusDegree = n; return p; }),
           py::arg("prime_bits"), py::arg("rotations"), py::arg("poly_modulus_degree"))
      .def_readonly("prime_bits", &CKKSParameters::primeBits)
      .def_readonly("rotations", &CKKSParameters::rotations)
      .def_readonly("poly_modulus_degree", &CKKSParameters::polyModulusDegree);
  py::class_<CKKSEncodingInfo>(mckks, "CKKSEncodingInfo")
      .def(py::init<Type, int, int>(), py::arg("input_type"), py::arg("scale"), py::arg("level"))
      .def_readonly("input_type", &CKKSEncodingInfo::inputType)
      .def_readonly("scale", &CKKSEncodingInfo::scale)
      .def_readonly("level", &CKKSEncodingInfo::level);
  py::class_<CKKSSignature>(mckks, "CKKSSignature")
      .def(py::init<int, std::map<std::string, CKKSEncodingInfo>>(), py::arg("vec_size"), py::arg("inputs"))
      .def_readonly("vec_size", &CKKSSignature::vecSize)
      .def_readonly("inputs", &CKKSSignature::inputs);

  py::module mb = m.def_submodule("_b200", "CUDA backend (replaces the reference's _seal submodule)");
  py::class_<B200Valuation>(mb, "B200Valuation", "A valuation for inputs or outputs holding encrypted values")
      .def(py::init<>())
      .def("names", [](const B200Valuation &v) { std::vector<std::string> n; for (auto &e : v) n.push_back(e.first); return n; })
      .def("set_cipher", [](B200Valuation &v, const std::string &name, const u64arr &data, double scale) {
        if (data.ndim() != 3) throw std::runtime_error("ciphertext array must be [size][ell][N]");
        HostCipher h; h.data = toHostBuf(data); h.size = (int)data.shape(0); h.ell = (int)data.shape(1); h.scale = scale;
        v[name] = std::move(h);
      }, "test/benchmark hook: inject a raw ciphertext [size][ell][N]")
      .def("set_seeded_cipher", [](B200Valuation &v, const std::string &name, const u64arr &c0, const py::bytes &seed, double scale) {
        if (c0.ndim() != 2) throw std::runtime_error("seeded ciphertext c0 must be [ell][N]");
        HostSeededCipher h; h.seed = toSeed(seed, "ciphertext"); h.c0 = toHostBuf(c0); h.ell = (int)c0.shape(0); h.scale = scale;
        v[name] = std::move(h);
      }, py::arg("name"), py::arg("c0"), py::arg("seed"), py::arg("scale"),
         "a seed-compressed fresh ciphertext (B200Secret.encrypt): c0 [ell][N] and the 32-byte seed from which c1 is expanded")
      .def("get_seed", [](const B200Valuation &v, const std::string &name) {
        auto *sc = std::get_if<HostSeededCipher>(&v.at(name));
        if (!sc) throw std::invalid_argument("value " + name + " is not a seeded ciphertext");
        return fromSeed(sc->seed);
      }, py::arg("name"), "the 32-byte seed of a seeded ciphertext")
      .def("set_plain", [](B200Valuation &v, const std::string &name, const u64arr &data, double scale) {
        if (data.ndim() != 2) throw std::runtime_error("plaintext array must be [ell][N]");
        HostPlain h; h.data = toHostBuf(data); h.ell = (int)data.shape(0); h.scale = scale; v[name] = std::move(h);
      })
      .def("set_raw", [](B200Valuation &v, const std::string &name, const std::vector<double> &x) { v[name] = std::make_shared<ConstantValue>(x.size(), x); })
      .def("get", [](const B200Valuation &v, const std::string &name) -> py::object {
        const SchemeValue &sv = v.at(name);
        if (auto *c = std::get_if<HostCipher>(&sv)) {
          const std::size_t N = c->data.size() / ((std::size_t)c->size * c->ell);
          u64arr a({(std::size_t)c->size, (std::size_t)c->ell, N});
          std::memcpy(a.mutable_data(), c->data.data(), c->data.size() * 8);
          return py::make_tuple("cipher", a, c->scale);
        }
        if (auto *p = std::get_if<HostPlain>(&sv)) {
          const std::size_t N = p->data.size() / (std::size_t)p->ell;
          u64arr a({(std::size_t)p->ell, N});
          std::memcpy(a.mutable_data(), p->data.data(), p->data.size() * 8);
          return py::make_tuple("plain", a, p->scale);
        }
        if (auto *sc = std::get_if<HostSeededCipher>(&sv)) {   // c0 only (the seed: get_seed)
          const std::size_t N = sc->c0.size() / (std::size_t)sc->ell;
          u64arr a({(std::size_t)sc->ell, N});
          std::memcpy(a.mutable_data(), sc->c0.data(), sc->c0.size() * 8);
          return py::make_tuple("seeded_cipher", a, sc->scale);
        }
        if (auto *r = std::get_if<StoredCipher>(&sv)) return py::make_tuple("stored", r->handle, py::none());
        if (auto *cc = std::get_if<HostCompactCipher>(&sv)) {
          const std::size_t W = cc->words.size() / 2;
          u64arr a({(std::size_t)2, W});
          std::memcpy(a.mutable_data(), cc->words.data(), cc->words.size() * 8);
          return py::make_tuple("compact_cipher", a, cc->scale);
        }
        return py::make_tuple("raw", std::get<std::shared_ptr<ConstantValue>>(sv)->values(), 0.0);
      })
      .def("set_stored", [](B200Valuation &v, const std::string &name, std::uint64_t handle) { v[name] = StoredCipher{handle}; },
           py::arg("name"), py::arg("handle"),
           "a reference to a ciphertext in a B200Server's store (B200Server.store returns the handles): the server stages the stored "
           "entry where this valuation would carry the ciphertext")
      .def("compact_bits", [](const B200Valuation &v, const std::string &name) {
        auto *cc = std::get_if<HostCompactCipher>(&v.at(name));
        if (!cc) throw std::invalid_argument("value " + name + " is not a compact ciphertext");
        return cc->bits;
      }, py::arg("name"), "the modulus bits b of a compact response")
      .def("set_compact_cipher", [](B200Valuation &v, const std::string &name, const u64arr &words, int bits, double scale) {
        if (bits < 1 || bits > 62) throw std::invalid_argument("compact ciphertext " + name + ": bits (" + std::to_string(bits) + ") must be in [1, 62]");
        if (words.ndim() != 2 || words.shape(0) != 2 || words.shape(1) < 1)
          throw std::invalid_argument("compact ciphertext " + name + ": words must be [2][W]");
        const std::size_t W = words.shape(1);
        // W = ceil(N bits / 64) for a power of two N: the smallest N it holds must be the largest too
        std::size_t N = 1;
        while ((N * 2 * bits + 63) / 64 <= W && N < ((std::size_t)1 << 20)) N *= 2;
        if ((N * bits + 63) / 64 != W) throw std::invalid_argument("compact ciphertext " + name + ": " + std::to_string(W) + " words per polynomial is not ceil(N bits / 64) for any N");
        HostCompactCipher h; h.words = toHostBuf(words); h.bits = bits; h.scale = scale;
        v[name] = std::move(h);
      }, py::arg("name"), py::arg("words"), py::arg("bits"), py::arg("scale"),
         "a compact response: words [2][ceil(N bits / 64)] (two bit-packed polynomials of N bits-bit fields), the compact scale");

  py::class_<PyPending, std::shared_ptr<PyPending>>(mb, "PendingBatch", "a submitted, not yet collected execute_batch");
  py::class_<B200Public> pub(mb, "B200Public", "The public part of the context: encryption and execution on the GPU");
  pub.def("encrypt", &B200Public::encrypt, py::arg("inputs"), py::arg("signature"))
      .def("execute", &B200Public::execute, py::arg("program"), py::arg("inputs"), py::call_guard<py::gil_scoped_release>())
      // the list is converted to pointers to the caller's valuations: no copy of the host ciphertexts
      .def("execute_full", [](B200Public &p, Program &prog, const B200Valuation &in) {
             std::vector<const B200Valuation *> v{&in};
             return std::move(p.executeMany(prog, v, 0)[0]);
           }, py::arg("program"), py::arg("inputs"), py::call_guard<py::gil_scoped_release>(),
           "execute() with full output ciphertexts whatever compact_outputs says (the sharded modes run their parts with it)")
      .def("execute_batch", [](B200Public &p, Program &prog, const std::vector<const B200Valuation *> &in) { return p.executeMany(prog, in); },
           py::arg("program"), py::arg("inputs"), py::call_guard<py::gil_scoped_release>(),
           "Execute one compiled program on a list of valuations with batched kernels; returns a list of valuations")
      // pipelined execute_batch: the handle keeps the program and the caller's valuations alive until it is collected
      .def("execute_batch_async", [](B200Public &p, py::object program, py::list inputs, int slot) {
             Program &prog = program.cast<Program &>();
             std::vector<const B200Valuation *> in;
             for (auto h : inputs) in.push_back(h.cast<const B200Valuation *>());
             auto out = std::make_shared<PyPending>();
             { py::gil_scoped_release rel; out->batch = p.submitMany(prog, in, slot); }
             out->program = program; out->inputs = inputs;
             return out;
           }, py::arg("program"), py::arg("inputs"), py::arg("slot") = 0,
           "Enqueue execute_batch (H2D, plan replays, D2H) and return a handle; collect with execute_batch_result(handle).  Batches in different slots (0..7) overlap")
      .def("execute_batch_result", [](B200Public &p, std::shared_ptr<PyPending> h) {
             std::vector<B200Valuation> outs;
             { py::gil_scoped_release rel; outs = p.collect(*h->batch); }
             return outs;
           }, py::arg("handle"))
      .def("set_input_sizes", [](B200Public &p, const std::map<std::string, int> &sizes) { p.options.inputSizes = sizes; },
           "ciphertext inputs that are not size 2 (name -> polynomials); applies to plans built afterwards")
      .def("drop_plan", &B200Public::dropExecutor, py::arg("program"), py::arg("batch") = 1, py::arg("replica") = 0)
      .def("plan_stats", [](B200Public &p, Program &prog, int batch, int replica) { return p.executorFor(prog, batch, replica).planStats(); },
           py::arg("program"), py::arg("batch") = 1, py::arg("replica") = 0, "shape of the execution plan: steps, hoist groups, rotation chunks, lazy rotation sums")
      .def("cipher_op_count", [](B200Public &p, Program &prog) { return p.executorFor(prog).cipherOpCount(); })
      // serialization (eva_b200/serialization.py): public key material only (never the secret key)
      .def("_export", [](B200Public &x) {
        auto s = x.shared();
        const std::size_t N = s->dev->N(), k = s->dev->k();
        py::dict d;
        d["N"] = N; d["primes"] = s->dev->primes();
        s->dev->sync();
        auto down = [&](const DBuf &b, std::vector<std::size_t> shape) {
          u64arr a(shape);
          s->dev->download(a.mutable_data(), b.get(), a.size() * 8);
          s->dev->sync();
          return a;
        };
        if (s->keys.pk) d["public_key"] = down(s->keys.pk, {2, k, N});
        if (s->keys.relin) d["relin_key"] = down(s->keys.relin, {k - 1, 2, k, N});
        py::dict g;
        for (auto &kv : s->keys.galois) g[py::int_(kv.first)] = down(kv.second, {k - 1, 2, k, N});
        d["galois_keys"] = g;
        // keys whose c1 rows are expanded from seeds: the seeds too (serialization then writes the compressed form)
        if (s->keys.relinSeed && s->keys.galoisSeeds.size() == s->keys.galois.size()) {
          d["relin_seed"] = fromSeed(*s->keys.relinSeed);
          py::dict gs;
          for (auto &kv : s->keys.galoisSeeds) gs[py::int_(kv.first)] = fromSeed(kv.second);
          d["galois_seeds"] = gs;
        }
        return d;
      })
      .def("launch_count", [](B200Public &p) { return evab_launch_count(p.shared()->dev->ctx()); })
      .def("primes", [](B200Public &p) { return p.shared()->dev->primes(); })
      // ---- benchmark hooks: device-resident execution on a caller-provided stream
      .def("stage_inputs", [](B200Public &p, Program &prog, const std::vector<const B200Valuation *> &in, std::uintptr_t stream, int replica) {
        Executor &ex = p.executorFor(prog, (int)in.size(), replica);
        p.checkStored(ex, prog, in.data(), nullptr, (int)in.size());   // rejects stored references: a context has no store
        p.stageInputs(ex, prog, in.data(), (int)in.size(), (void *)stream);
      }, py::arg("program"), py::arg("inputs"), py::arg("stream"), py::arg("replica") = 0)
      .def("run_resident", [](B200Public &p, Program &prog, std::uintptr_t stream, int batch, int replica) { p.executorFor(prog, batch, replica).run((void *)stream); },
           py::arg("program"), py::arg("stream"), py::arg("batch") = 1, py::arg("replica") = 0, py::call_guard<py::gil_scoped_release>())
      .def("sync", [](B200Public &p, std::uintptr_t stream) { p.shared()->dev->sync((void *)stream); }, py::call_guard<py::gil_scoped_release>())
      // ---- device-resident plumbing of the DAG-sharded mode (eva_b200/shard.py): where a plan keeps its named
      // inputs and outputs in device memory, so that NCCL can gather partial ciphertexts straight from one
      // rank's arena into another's (no host staging), and a download of the outputs of a resident run
      .def("io_pointers", [](B200Public &p, Program &prog, int batch, int replica) {
        Executor &ex = p.executorFor(prog, batch, replica);
        const std::size_t N = p.shared()->dev->N();
        auto describe = [&](const Term::Ptr &t) -> py::object {
          const ValueInfo &vi = ex.info(t);
          if (vi.kind != Kind::Cipher && vi.kind != Kind::Plain) return py::none();
          const std::size_t polys = vi.kind == Kind::Cipher ? (std::size_t)vi.size : 1;
          py::dict d;
          d["ptr"] = (std::uintptr_t)ex.valuePtr(t, 0); d["bytes"] = polys * (std::size_t)vi.ell * N * 8;
          d["size"] = (int)polys; d["ell"] = vi.ell; d["scale"] = vi.scale; d["cipher"] = vi.kind == Kind::Cipher;
          return d;
        };
        py::dict ins, outs;
        for (auto &in : prog.getInputs()) ins[py::str(in.first)] = describe(in.second);
        for (auto &o : prog.getOutputs()) outs[py::str(o.first)] = describe(o.second);
        py::dict r; r["inputs"] = ins; r["outputs"] = outs;
        return r;
      }, py::arg("program"), py::arg("batch") = 1, py::arg("replica") = 0)
      .def("download_outputs", [](B200Public &p, Program &prog, std::uintptr_t stream, int replica) {
        Executor &ex = p.executorFor(prog, 1, replica);
        auto dev = p.shared()->dev;
        const std::size_t N = dev->N();
        B200Valuation out;
        for (auto &o : prog.getOutputs()) {
          const ValueInfo &vi = ex.info(o.second);
          if (vi.kind == Kind::Cipher) {
            HostCipher h; h.size = vi.size; h.ell = vi.ell; h.scale = vi.scale; h.data.resize((std::size_t)vi.size * vi.ell * N);
            dev->download(h.data.data(), ex.valuePtr(o.second, 0), h.data.size() * 8, (void *)stream);
            out[o.first] = std::move(h);
          } else if (vi.kind == Kind::Plain) {
            HostPlain h; h.ell = vi.ell; h.scale = vi.scale; h.data.resize((std::size_t)vi.ell * N);
            dev->download(h.data.data(), ex.valuePtr(o.second, 0), h.data.size() * 8, (void *)stream);
            out[o.first] = std::move(h);
          } else {
            out[o.first] = std::make_shared<ConstantValue>(prog.getVecSize(), ex.rawValue(o.second->index, 0));
          }
        }
        dev->sync((void *)stream);
        if (ex.flagsRaised())
          throw std::runtime_error("a digit of a rotated ciphertext held a zero coefficient: rerun with set_options(hoist_mod_up=False) (execute() does so by itself)");
        return out;
      }, py::arg("program"), py::arg("stream"), py::arg("replica") = 0, py::call_guard<py::gil_scoped_release>())
      // ---- test hooks
      .def("debug_value", &debugValue, py::arg("program"), py::arg("index"), py::arg("batch") = 1, py::arg("instance") = 0)
      .def("encode", [](B200Public &p, const std::vector<double> &values, double scale, int ell, bool host) {
        auto dev = p.shared()->dev;
        DBuf pt(dev, (std::size_t)ell * dev->N());
        std::vector<double> rep;
        const std::size_t slots = dev->N() / 2;
        for (std::size_t r = slots / values.size(); r > 0; --r) rep.insert(rep.end(), values.begin(), values.end());
        if (host) p.shared()->client->encoder().encodeHost(rep, scale, ell, pt.get());
        else p.shared()->client->encoder().encode(values, scale, ell, pt.get());
        u64arr a({(std::size_t)ell, (std::size_t)dev->N()});
        dev->download(a.mutable_data(), pt.get(), a.size() * 8);
        dev->sync();
        return a;
      }, py::arg("values"), py::arg("scale"), py::arg("ell"), py::arg("host") = false)
      // test hook: Encryptor::encrypt of a plaintext polynomial [ell][N] with EXPLICIT randomness -> ciphertext [2][ell][N]
      .def("encrypt_poly", [](B200Public &p, const u64arr &pt, const std::vector<int> &u, const std::vector<int> &e0, const std::vector<int> &e1) {
        auto s = p.shared();
        if (!s->keys.pk) throw std::runtime_error("this context has no public key");
        if (pt.ndim() != 2 || (std::size_t)pt.shape(1) != s->dev->N()) throw std::runtime_error("plaintext array must be [ell][N]");
        const int ell = (int)pt.shape(0);
        DBuf d(s->dev, pt.size());
        s->dev->upload(d.get(), pt.data(), pt.size() * 8);
        DBuf ct = s->client->encryptWith(s->keys, d.get(), ell, u, e0, e1);
        u64arr a({(std::size_t)2, (std::size_t)ell, (std::size_t)s->dev->N()});
        s->dev->download(a.mutable_data(), ct.get(), a.size() * 8);
        s->dev->sync();
        return a;
      }, py::arg("plaintext"), py::arg("u"), py::arg("e0"), py::arg("e1"))
      .def("encrypt_seeded_poly", [](B200Public &p, const u64arr &pt, const py::bytes &seed, const std::vector<int> &e) {
        return encryptSeededPoly(p.shared(), pt, seed, e);
      }, py::arg("plaintext"), py::arg("seed"), py::arg("e"), "test hook (contexts that hold the secret key): secret-key encryption with an explicit seed and error")
      .def("decode", [](B200Public &p, const u64arr &pt, double scale) {
        auto dev = p.shared()->dev;
        DBuf d(dev, pt.size());
        dev->upload(d.get(), pt.data(), pt.size() * 8);
        return p.shared()->client->encoder().decode(d.get(), (int)pt.shape(0), scale);
      });
  defSetOptions(pub);
  py::class_<B200Secret>(mb, "B200Secret","The secret part of the context: decryption, and secret-key encryption of compact inputs")
      .def("decrypt", &B200Secret::decrypt, py::arg("enc_outputs"), py::arg("signature"))
      .def("encrypt", &B200Secret::encrypt, py::arg("inputs"), py::arg("signature"),
           "B200Public.encrypt with the secret key: every Cipher input becomes a seeded ciphertext (c0 and a 32-byte seed, half the bytes); "
           "Plain and Raw inputs as B200Public.encrypt makes them")
      .def("encrypt_seeded_poly", [](B200Secret &x, const u64arr &pt, const py::bytes &seed, const std::vector<int> &e) {
        return encryptSeededPoly(x.shared(), pt, seed, e);
      }, py::arg("plaintext"), py::arg("seed"), py::arg("e"), "test hook: secret-key encryption with an explicit seed and error -> [2][ell][N]")
      // test hook: Decryptor::decrypt of a raw ciphertext [size][ell][N] -> plaintext polynomial [ell][N] (before decoding)
      .def("decrypt_poly", [](B200Secret &x, const u64arr &ct) {
        auto s = x.shared();
        if (ct.ndim() != 3 || (std::size_t)ct.shape(2) != s->dev->N()) throw std::runtime_error("ciphertext array must be [size][ell][N]");
        DBuf d(s->dev, ct.size());
        s->dev->upload(d.get(), ct.data(), ct.size() * 8);
        DBuf pt = s->client->decrypt(s->keys, d.get(), (int)ct.shape(0), (int)ct.shape(1));
        u64arr a({(std::size_t)ct.shape(1), (std::size_t)s->dev->N()});
        s->dev->download(a.mutable_data(), pt.get(), a.size() * 8);
        s->dev->sync();
        return a;
      }, py::arg("ciphertext"))
      // test hook: the centred integers z = (y0 + y1 s) mod 2^bits of a compact ciphertext [2][W], before decoding
      .def("decrypt_compact_poly", [](B200Secret &x, const u64arr &words, int bits) {
        if (words.ndim() != 2 || words.shape(0) != 2) throw std::invalid_argument("compact ciphertext words must be [2][W]");
        HostCompactCipher h; h.words = toHostBuf(words); h.bits = bits; h.scale = 1.0;
        std::vector<std::int64_t> z;
        x.decryptCompact(h, "compact ciphertext", &z);
        py::array_t<std::int64_t> a(z.size());
        std::memcpy(a.mutable_data(), z.data(), z.size() * 8);
        return a;
      }, py::arg("words"), py::arg("bits"))
      .def("decode", [](B200Secret &x, const u64arr &pt, double scale) {
        auto s = x.shared();
        DBuf d(s->dev, pt.size());
        s->dev->upload(d.get(), pt.data(), pt.size() * 8);
        return s->client->encoder().decode(d.get(), (int)pt.shape(0), scale);
      }, py::arg("plaintext"), py::arg("scale"))
      // serialization (eva_b200/serialization.py): secret key image [k][N] + the modulus chain
      .def("_export", [](B200Secret &x) {
        auto s = x.shared();
        py::dict d;
        d["N"] = s->dev->N(); d["primes"] = s->dev->primes();
        u64arr a({(std::size_t)s->dev->k(), (std::size_t)s->dev->N()});
        s->dev->sync();
        s->dev->download(a.mutable_data(), s->keys.sk.get(), a.size() * 8);
        s->dev->sync();
        d["secret_key"] = a;
        return d;
      });

  // ---- multi-tenant serving: one device, one parameter set, the evaluation keys of many clients in a key bank
  typedef std::vector<std::pair<int, const B200Valuation *>> Requests;
  py::class_<B200Server> srv(mb, "B200Server",
                             "Executes compiled programs for many clients: each client's evaluation keys are a tenant of a key bank of fixed "
                             "capacity, the plans are shared by all tenants, and every instance of a batch runs with its own tenant's keys");
  srv.def(py::init([](const CKKSParameters &params, int capacity, int device, std::optional<int> maxTenants, const std::string &rotationKeys,
                       const std::string &hoistConstants, const std::string &keyStorage, int c1Cache, int storeEntries, std::optional<int> maxStored,
                       const std::string &storeStorage) {
        return std::make_unique<B200Server>(params, capacity, device, maxTenants ? *maxTenants : -1, rotationKeys, hoistConstants, keyStorage, c1Cache,
                                            storeEntries, maxStored ? *maxStored : -1, storeStorage);
      }), py::arg("params"), py::arg("capacity") = 64, py::arg("device") = 0, py::arg("max_tenants") = py::none(), py::arg("rotation_keys") = "program",
      py::arg("hoist_constants") = "stored", py::arg("key_storage") = "expanded", py::arg("c1_cache") = 0, py::arg("store_entries") = 0,
      py::arg("max_stored") = py::none(), py::arg("store_storage") = "expanded",
      "capacity: device slots (key-bank regions).  max_tenants None or == capacity: a tenant id is its slot, filled when its keys are "
      "added.  max_tenants > capacity: up to max_tenants tenants' keys in page-locked host memory, paged into the slots (least "
      "recently used first) as batches need them.  rotation_keys: the Galois keys every tenant supplies -- \"program\", one per "
      "rotation step of the program; \"power_of_two\", one per NAF term of its steps (the other rotations are composed from them, "
      "as SEAL's rotate_vector does).  hoist_constants: \"stored\", every slot also holds the hoist constants of its Galois keys "
      "(computed at every fill); \"inline\", slots hold the keys only and the hoisted rotations form the constants inside the "
      "key-switch inner product (same outputs, smaller slots; approx_hoist is not available).  key_storage: \"expanded\", every key in "
      "full; \"seeded\" (with hoist_constants=\"inline\"), slots hold each key's c0 rows and seed and the key switches draw the uniform "
      "half from the seed (same outputs, half the slot; compressed keys only).  c1_cache (key_storage=\"seeded\", 0 <= c1_cache <= "
      "capacity): device regions, each holding the expanded c1 rows of one tenant; the instances of a batch whose tenant holds one read "
      "them instead of drawing (same outputs).  The tenants with the most instances in a batch are admitted first, the least recently "
      "used region is evicted; tenants without a region draw.  store_entries: device entries of the ciphertext store, each holding "
      "one stored size-2 input ciphertext (store / release; 0: no store).  max_stored None or == store_entries: every stored "
      "ciphertext holds a device entry.  max_stored > store_entries: up to max_stored stored ciphertexts in page-locked host memory, "
      "paged into the device entries (least recently used first) as batches name them; a batch names at most store_entries "
      "distinct ones.  store_storage: \"expanded\", device entries hold whole ciphertexts (a seeded one is expanded when it is "
      "written to the device); \"seeded\", seeded ciphertexts only (B200Secret.encrypt), entries hold c0 rows and the seed and "
      "staging draws the uniform half (same outputs, half the entry)")
      .def("add_raw_keys", [](B200Server &s, const u64arr &relin, const std::map<u64, u64arr> &galois) {
        const std::size_t kk = s.shared()->dev->k(), N = s.shared()->dev->N();
        requireShape(relin, {kk - 1, 2, kk, N}, "relinearization key");
        std::map<u64, const u64 *> g;   // the elements of the rotation set (addKeys reports a missing one)
        for (u64 e : s.bank().elements())
          if (auto it = galois.find(e); it != galois.end()) {
            requireShape(it->second, {kk - 1, 2, kk, N}, "Galois key");
            g[e] = it->second.data();
          }
        py::gil_scoped_release rel;
        return s.addKeys(relin.data(), g);
      }, py::arg("relin_key"), py::arg("galois_keys"), "copy a client's relinearization key and Galois keys (host arrays [k-1][2][k][N]) into a "
         "free tenant slot and compute its hoist constants (with paging: into page-locked host memory, no device work); returns the tenant id")
      .def("add_compressed_keys", [](B200Server &s, const u64arr &relinC0, const py::bytes &relinSeed, const std::map<u64, u64arr> &galoisC0,
                                     const std::map<u64, py::bytes> &galoisSeeds) {
        const std::size_t kk = s.shared()->dev->k(), N = s.shared()->dev->N();
        requireShape(relinC0, {kk - 1, kk, N}, "compressed relinearization key");
        const KeySeed rs = toSeed(relinSeed, "relinearization key");
        std::map<u64, std::pair<const u64 *, KeySeed>> g;   // the elements of the rotation set (addCompressedKeys reports a missing one)
        for (u64 e : s.bank().elements()) {
          auto it = galoisC0.find(e);
          if (it == galoisC0.end()) continue;
          requireShape(it->second, {kk - 1, kk, N}, "compressed Galois key");
          auto sd = galoisSeeds.find(e);
          if (sd == galoisSeeds.end()) throw std::invalid_argument("no seed for the Galois key of element " + std::to_string(e));
          g[e] = {it->second.data(), toSeed(sd->second, "Galois key")};
        }
        py::gil_scoped_release rel;
        return s.addCompressedKeys(relinC0.data(), rs, g);
      }, py::arg("relin_c0"), py::arg("relin_seed"), py::arg("galois_c0"), py::arg("galois_seeds"),
         "add a client's keys in compressed form: the c0 rows (host arrays [k-1][k][N]) and the 32-byte seed of the relinearization key "
         "and of every Galois key; the c1 rows are expanded on the device (with paging: the compressed form is what the host store keeps, "
         "half the bytes of add_raw_keys).  Returns the tenant id")
      .def("add_keys", [](B200Server &s, B200Public &p) {
        auto src = p.shared();
        if (src->dev->N() != s.shared()->dev->N() || src->dev->primes() != s.shared()->dev->primes())
          throw std::invalid_argument("the context's N / primes do not match the server's");
        const std::size_t kk = s.shared()->dev->k(), kN = kk * s.shared()->dev->N(), words = (kk - 1) * 2 * kN;
        if (!src->keys.relin || src->keys.relin.words() != words) throw std::invalid_argument("the context has no relinearization key of the server's shape");
        // keys expanded from seeds travel compressed: only their c0 rows are read back
        bool seeded = src->keys.relinSeed.has_value();
        for (u64 e : s.bank().elements())
          if (src->keys.galois.count(e) && !src->keys.galoisSeeds.count(e)) seeded = false;
        const std::size_t hw = seeded ? words / 2 : words;
        auto fetch = [&](const DBuf &key, std::vector<u64> &h) {
          h.resize(hw);
          if (!seeded) { src->dev->download(h.data(), key.get(), words * 8); return; }
          for (std::size_t J = 0; J + 1 < kk; J++) src->dev->download(h.data() + J * kN, key.get() + J * 2 * kN, kN * 8);
        };
        std::vector<u64> relin;
        std::map<u64, std::vector<u64>> gal;
        src->dev->sync();
        fetch(src->keys.relin, relin);
        for (u64 e : s.bank().elements()) {
          auto it = src->keys.galois.find(e);
          if (it == src->keys.galois.end()) continue;   // addKeys / addCompressedKeys report it
          if (it->second.words() != words) throw std::invalid_argument("Galois key does not match the server's shape");
          fetch(it->second, gal[e]);
        }
        src->dev->sync();
        py::gil_scoped_release rel;
        if (seeded) {
          std::map<u64, std::pair<const u64 *, KeySeed>> g;
          for (auto &kv : gal) g[kv.first] = {kv.second.data(), src->keys.galoisSeeds.at(kv.first)};
          return s.addCompressedKeys(relin.data(), *src->keys.relinSeed, g);
        }
        std::map<u64, const u64 *> g;
        for (auto &kv : gal) g[kv.first] = kv.second.data();
        return s.addKeys(relin.data(), g);
      }, py::arg("public_context"), "add a client's B200Public (same N and primes): compressed (add_compressed_keys) when its keys were "
         "expanded from seeds (generate_keys, or a loaded compressed context), in full (add_raw_keys) otherwise")
      .def("remove_keys", &B200Server::removeKeys, py::arg("tenant"), "also releases the tenant's stored ciphertexts")
      .def("store", &B200Server::store, py::arg("tenant"), py::arg("enc"), py::call_guard<py::gil_scoped_release>(),
           "keep the ciphertexts of `enc` (B200Public.encrypt or B200Secret.encrypt; every value a ciphertext; with "
           "store_storage=\"seeded\" B200Secret.encrypt only) as the tenant's entries, all or nothing: on the device (with "
           "store_storage=\"expanded\" a seeded one is expanded once here), or with max_stored > store_entries in page-locked host "
           "memory only, a seeded one as c0 rows and seed.  Returns {name: handle}: a request names an entry with "
           "B200Valuation.set_stored(name, handle), and its outputs are those of the same ciphertext sent inline")
      .def("release", &B200Server::release, py::arg("handle"), "free a stored ciphertext's entry; its handle names nothing afterwards")
      .def("execute", [](B200Server &s, Program &prog, int tenant, const B200Valuation &in) {
        return std::move(s.executeBatch(prog, {{tenant, &in}})[0]);
      }, py::arg("program"), py::arg("tenant"), py::arg("inputs"), py::call_guard<py::gil_scoped_release>())
      .def("execute_batch", &B200Server::executeBatch, py::arg("program"), py::arg("requests"), py::call_guard<py::gil_scoped_release>(),
           "requests: [(tenant, valuation), ...]; returns a list of valuations")
      .def("execute_batch_async", [](B200Server &s, py::object program, py::list requests, int slot) {
        Program &prog = program.cast<Program &>();
        Requests rq = requests.cast<Requests>();
        auto out = std::make_shared<PyPending>();
        { py::gil_scoped_release rel; out->batch = s.submit(prog, rq, slot); }
        out->program = program; out->inputs = requests;
        return out;
      }, py::arg("program"), py::arg("requests"), py::arg("slot") = 0)
      .def("execute_batch_result", [](B200Server &s, std::shared_ptr<PyPending> h) {
        std::vector<B200Valuation> outs;
        { py::gil_scoped_release rel; outs = s.pub().collect(*h->batch); }
        return outs;
      }, py::arg("handle"))
      .def("drop_plan", [](B200Server &s, Program &prog, int batch, int replica) { s.pub().dropExecutor(prog, batch, replica); },
           py::arg("program"), py::arg("batch") = 1, py::arg("replica") = 0)
      .def("plan_stats", [](B200Server &s, Program &prog, int batch, int replica) { return s.pub().executorFor(prog, batch, replica).planStats(); },
           py::arg("program"), py::arg("batch") = 1, py::arg("replica") = 0)
      .def("plans_built", [](B200Server &s) { return s.pub().plansBuilt; }, "plans built so far (each: plan, arena, graph capture)")
      .def("launch_count", [](B200Server &s) { return evab_launch_count(s.shared()->dev->ctx()); })
      .def("bank_info", [](B200Server &s) {
        const KeyBank &b = s.bank();
        std::lock_guard<std::mutex> guard(s.shared()->execMutex);   // add / remove change the occupancy under it
        const KeyPager *pg = s.shared()->pager.get();
        py::dict d;
        d["capacity"] = b.capacity(); d["tenants"] = pg ? pg->tenants() : b.tenants(); d["galois_elements"] = b.elements();
        d["tenant_bytes"] = b.stride() * 8; d["key_bytes_per_tenant"] = b.keyWords() * 8; d["hoist_const_bytes_per_tenant"] = b.constWords() * 8;
        d["bank_bytes"] = b.stride() * 8 * (std::size_t)b.capacity();
        d["device_slots"] = b.capacity();
        d["max_tenants"] = pg ? pg->maxTenants() : b.capacity();
        std::vector<int> resident;
        if (pg) resident = pg->cache().holders();
        else for (int t = 0; t < b.capacity(); t++) if (b.occupied(t)) resident.push_back(t);
        d["resident"] = resident;
        d["host_key_bytes"] = pg ? pg->hostBytes() : 0;
        d["compressed_tenants"] = pg ? pg->compressedTenants() : b.compressedTenants();
        d["fills"] = b.fills();
        d["evictions"] = pg ? pg->cache().evictions() : 0;
        d["rotation_keys"] = s.rotationKeys();
        d["hoist_constants"] = s.hoistConstants();
        d["key_storage"] = s.keyStorage();
        d["indicator_bytes"] = b.indicatorBytes();
        const C1Store *c1 = s.shared()->c1.get();
        d["c1_cache"] = b.c1Regions();
        d["c1_cache_bytes"] = b.stride() * 8 * (std::size_t)b.c1Regions();
        d["c1_cached"] = c1 ? c1->cache().holders() : std::vector<int>();
        d["c1_fills"] = c1 ? c1->cache().fills() : 0;
        d["c1_evictions"] = c1 ? c1->cache().evictions() : 0;
        const CipherStore *st = s.cipherStore();
        const std::size_t entryBytes = CipherStore::entryWords(s.shared()->dev->k(), s.shared()->dev->N(), CipherStore::seededLayout(s.storeStorage())) * 8;
        d["store_entries"] = st ? st->capacity() : 0;
        d["max_stored"] = st ? st->maxStored() : 0;
        d["store_storage"] = s.storeStorage();
        d["stored"] = st ? st->used() : 0;
        d["store_resident"] = st ? st->resident() : std::vector<std::uint64_t>();
        d["store_fills"] = st ? st->fills() : 0;
        d["store_evictions"] = st ? st->evictions() : 0;
        d["store_host_bytes"] = st ? st->hostBytes() : 0;
        d["store_entry_bytes"] = entryBytes;
        d["store_bytes"] = st ? entryBytes * (std::size_t)st->capacity() : 0;
        return d;
      }, "capacity / device_slots: key-bank regions; rotation_keys: the key set of galois_elements (\"program\" or \"power_of_two\"); "
         "hoist_constants: \"stored\" or \"inline\" (then hoist_const_bytes_per_tenant is 0 and indicator_bytes the one shared copy of "
         "the elements' indicator rows); key_storage: \"expanded\" or \"seeded\" (key_bytes_per_tenant then counts c0 rows and seeds); "
         "max_tenants: tenant ids (more than the slots: paging); resident: the tenants "
         "holding a slot; host_key_bytes: page-locked host memory of the paged keys (compressed tenants: c0 rows and seeds); "
         "compressed_tenants: tenants added in compressed form; fills: slots filled (keys uploaded and "
         "constants computed); evictions: resident tenants displaced by a fill; c1_cache: c1 regions (c1_cache_bytes of device memory); "
         "c1_cached: the tenants holding one; c1_fills: regions expanded; c1_evictions: cached tenants displaced by a fill; "
         "store_entries: device entries of the ciphertext store (store_bytes of device memory, store_entry_bytes each: 2 (k-1) N words "
         "with store_storage \"expanded\", (k-1) N with \"seeded\"); max_stored: stored ciphertexts it can hold (more than "
         "store_entries: paging); stored: entries in use; store_resident: the handles holding a device entry; store_fills: device "
         "entries written from host memory (paging); store_evictions: resident entries displaced by a fill; store_host_bytes: "
         "page-locked host memory of the paged entries (2 ell N words each, ell N for a seeded ciphertext, whose seed is kept "
         "beside them)")
      .def("primes", [](B200Server &s) { return s.shared()->dev->primes(); })
      // ---- benchmark hooks (as B200Public's): device-resident execution of requests staged on a plan replica
      .def("stage_inputs", [](B200Server &s, Program &prog, const Requests &rq, std::uintptr_t stream, int replica) {
        s.stageInputs(prog, rq, (void *)stream, replica);
      }, py::arg("program"), py::arg("requests"), py::arg("stream"), py::arg("replica") = 0)
      .def("run_resident", [](B200Server &s, Program &prog, std::uintptr_t stream, int batch, int replica, const std::vector<int> &tenants) {
        s.runResident(prog, (void *)stream, batch, replica, tenants);
      }, py::arg("program"), py::arg("stream"), py::arg("batch") = 1, py::arg("replica") = 0, py::arg("tenants") = std::vector<int>(),
         py::call_guard<py::gil_scoped_release>(),
         "tenants: replace the staged tenants of the replica (with paging, missing ones are filled before the run)")
      .def("debug_value", [](B200Server &s, Program &prog, std::uint64_t index, int batch, int b) { return debugValue(s.pub(), prog, index, batch, b); },
           py::arg("program"), py::arg("index"), py::arg("batch") = 1, py::arg("instance") = 0);
  defSetOptions(srv);

  mb.def("generate_keys", [](const CKKSParameters &p, int device, std::uint64_t seed, const std::string &rotationKeys) {
           return generateKeys(p, device, seed, rotationKeys);
         }, py::arg("abstract_params"), py::arg("device") = 0, py::arg("seed") = 0, py::arg("rotation_keys") = "program",
         "rotation_keys: \"program\" -- a Galois key for every rotation step of the program; \"power_of_two\" -- one for every NAF term "
         "of its nonzero steps (but +-N/2), ascending, from which every rotation of the program is composed as SEAL's rotate_vector does");
  // test/benchmark hook: evaluation context from externally supplied key material
  mb.def("context_from_raw_keys", [](std::uint64_t N, const std::vector<u64> &primes, const u64arr &relin, const std::map<u64, u64arr> &galois, int device) {
    auto s = std::make_shared<Shared>();
    s->dev = std::make_shared<Device>(N, primes, device);
    s->client = std::make_unique<CkksClient>(s->dev, 0);   // evaluation context; any encryption through it draws OS entropy
    const std::size_t kk = primes.size();
    requireShape(relin, {kk - 1, 2, kk, (std::size_t)N}, "relinearization key");
    for (auto &g : galois) requireShape(g.second, {kk - 1, 2, kk, (std::size_t)N}, "Galois key");
    s->keys.relin = DBuf(s->dev, relin.size());
    s->dev->upload(s->keys.relin.get(), relin.data(), relin.size() * 8);
    for (auto &g : galois) {
      check(evab_galois_prepare(s->dev->ctx(), g.first));
      DBuf d(s->dev, g.second.size());
      s->dev->upload(d.get(), g.second.data(), g.second.size() * 8);
      s->keys.galois.emplace(g.first, std::move(d));
    }
    s->dev->sync();
    return std::make_unique<B200Public>(s);
  }, py::arg("N"), py::arg("primes"), py::arg("relin_key"), py::arg("galois_keys"), py::arg("device") = 0);
  // serialization: contexts rebuilt from saved key material
  // relin_seed / galois_seeds: the matching keys are compressed -- c0 rows [k-1][k][N] -- and their c1 rows are expanded on the device
  mb.def("public_from_raw", [](std::uint64_t N, const std::vector<u64> &primes, py::object pk, py::object relin, const std::map<u64, u64arr> &galois, int device,
                               py::object relinSeed, const std::map<u64, py::bytes> &galoisSeeds) {
    auto s = std::make_shared<Shared>();
    s->dev = std::make_shared<Device>(N, primes, device);
    s->client = std::make_unique<CkksClient>(s->dev, 0);   // OS entropy (csprng.hpp)
    auto up = [&](DBuf &dst, const u64arr &a) { dst = DBuf(s->dev, a.size()); s->dev->upload(dst.get(), a.data(), a.size() * 8); s->dev->sync(); };
    const std::size_t kk = primes.size();
    for (auto &g : galoisSeeds) if (!galois.count(g.first)) throw std::invalid_argument("a Galois seed without its key");
    if (!pk.is_none()) { requireShape(py::cast<u64arr>(pk), {2, kk, (std::size_t)N}, "public key"); up(s->keys.pk, py::cast<u64arr>(pk)); }
    if (!relin.is_none()) {
      const u64arr r = py::cast<u64arr>(relin);
      if (relinSeed.is_none()) { requireShape(r, {kk - 1, 2, kk, (std::size_t)N}, "relinearization key"); up(s->keys.relin, r); }
      else {
        requireShape(r, {kk - 1, kk, (std::size_t)N}, "compressed relinearization key");
        s->keys.relinSeed = toSeed(py::cast<py::bytes>(relinSeed), "relinearization key");
        s->keys.relin = expandCompressedKey(s->dev, r.data(), *s->keys.relinSeed);
      }
    }
    for (auto &g : galois) {
      if (galoisSeeds.count(g.first)) requireShape(g.second, {kk - 1, kk, (std::size_t)N}, "compressed Galois key");
      else requireShape(g.second, {kk - 1, 2, kk, (std::size_t)N}, "Galois key");
    }
    for (auto &g : galois) {
      check(evab_galois_prepare(s->dev->ctx(), g.first));
      DBuf d;
      if (auto sd = galoisSeeds.find(g.first); sd != galoisSeeds.end()) {
        const KeySeed seed = toSeed(sd->second, "Galois key");
        s->keys.galoisSeeds[g.first] = seed;
        d = expandCompressedKey(s->dev, g.second.data(), seed);
      } else {
        up(d, g.second);
      }
      s->keys.galois.emplace(g.first, std::move(d));
    }
    return std::make_unique<B200Public>(s);
  }, py::arg("N"), py::arg("primes"), py::arg("public_key"), py::arg("relin_key"), py::arg("galois_keys"), py::arg("device") = 0,
     py::arg("relin_seed") = py::none(), py::arg("galois_seeds") = std::map<u64, py::bytes>());
  mb.def("secret_from_raw", [](std::uint64_t N, const std::vector<u64> &primes, const u64arr &sk, int device) {
    auto s = std::make_shared<Shared>();
    s->dev = std::make_shared<Device>(N, primes, device);
    s->client = std::make_unique<CkksClient>(s->dev, 0);
    requireShape(sk, {primes.size(), (std::size_t)N}, "secret key");
    s->keys.sk = DBuf(s->dev, sk.size());
    s->dev->upload(s->keys.sk.get(), sk.data(), sk.size() * 8);
    s->dev->sync();
    return std::make_unique<B200Secret>(s);
  }, py::arg("N"), py::arg("primes"), py::arg("secret_key"), py::arg("device") = 0);
  mb.def("create_coeff_modulus", [](std::uint64_t N, const std::vector<int> &bits) { return hmod::createCoeffModulus(N, bits); });
}
