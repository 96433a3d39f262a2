// ckks_client.hpp -- client side of the backend: CKKS encoder/decoder (FP64
// canonical-embedding FFT on the host, NTTs on the device), key generation,
// public-key encryption and decryption.  Replaces what the reference obtains
// from seal::CKKSEncoder / KeyGenerator / Encryptor / Decryptor at
// eva/seal/seal.cpp:24-102,124-146,174-203 and seal_executor.h:217-243
// (SURVEY.md Appendix A.9-A.11).  All polynomial arithmetic runs on the GPU
// through the C-ABI, and so do the encoder's and the decoder's FP64 transforms; only the sampling is host code.
#pragma once
#include "runtime.hpp"
#include <array>
#include <cmath>
#include <optional>
#include <random>
#include "csprng.hpp"

namespace evab {

class CkksEncoder {
public:
  explicit CkksEncoder(std::shared_ptr<Device> dev) : dev_(std::move(dev)), N_(dev_->N()) {
    logN_ = 0;
    while ((u64(1) << logN_) < N_) logN_++;
    const u64 m = 2 * N_, slots = N_ / 2;
    rootRe_.resize(N_); rootIm_.resize(N_);
    for (u64 i = 0; i < N_; i++) unitRoot(bitrev(i), m, rootRe_[i], rootIm_[i]);
    slotIndex_.resize(N_);
    u64 pos = 1;
    for (u64 i = 0; i < slots; i++) {  // 3^i orbit of the 2N-th roots
      slotIndex_[i] = (std::uint32_t)bitrev((pos - 1) >> 1);
      slotIndex_[slots | i] = (std::uint32_t)bitrev((m - pos - 1) >> 1);
      pos = (pos * 3) & (m - 1);
    }
  }
  u64 slotCount() const { return N_ / 2; }

  // values (<= N/2 of them, zero padded) -> coefficient residues [ell][N] (NOT yet NTT'd)
  void embed(const std::vector<double> &values, double scale, int ell, std::vector<u64> &out) const {
    const u64 slots = N_ / 2;
    if (values.size() > slots) throw std::invalid_argument("values_size is too large");
    std::vector<double> re(N_, 0.0), im(N_, 0.0);
    for (std::size_t i = 0; i < values.size(); i++) {
      re[slotIndex_[i]] = values[i];
      re[slotIndex_[slots + i]] = values[i];
    }
    // inverse special FFT: Gentleman-Sande from bit-reversed order with conjugate twiddles
    u64 gap = 1;
    for (u64 m = N_ >> 1; m >= 1; m >>= 1) {
      for (u64 i = 0; i < m; i++) {
        const double wr = rootRe_[m + i], wi = -rootIm_[m + i];
        const u64 base = 2 * i * gap;
        for (u64 j = base; j < base + gap; j++) {
          const double ur = re[j], ui = im[j], vr = re[j + gap], vi = im[j + gap];
          re[j] = ur + vr; im[j] = ui + vi;
          const double dr = ur - vr, di = ui - vi;
          re[j + gap] = dr * wr - di * wi;
          im[j + gap] = dr * wi + di * wr;
        }
      }
      gap <<= 1;
    }
    const double fix = scale / (double)N_;
    const auto &P = dev_->primes();
    out.assign((std::size_t)ell * N_, 0);
    for (u64 j = 0; j < N_; j++) {
      const double c = std::round(re[j] * fix);
      const bool neg = std::signbit(c);
      const double mag = std::fabs(c);
      u64 mant; int sh = 0;
      if (mag < 18446744073709551616.0) mant = (u64)mag;
      else { int ex; const double fr = std::frexp(mag, &ex); mant = (u64)std::ldexp(fr, 64); sh = ex - 64; }  // mag = mant * 2^sh exactly
      for (int i = 0; i < ell; i++) {
        const u64 p = P[i];
        u64 v = mant % p;
        if (sh) v = hmod::mul(v, hmod::pow(2, (u64)sh, p), p);
        out[(std::size_t)i * N_ + j] = (neg && v) ? p - v : v;
      }
    }
  }
  // encode into device memory d_pt[ell][N] in NTT form (seal::CKKSEncoder::encode)
  // device path: the batched encoder kernels behind evab_encode (FP64 FFT + NTT on the GPU)
  void encode(const std::vector<double> &values, double scale, int ell, u64 *d_pt, void *stream = nullptr) const {
    if (values.empty() || (N_ / 2) % values.size()) throw std::invalid_argument("values size must divide the slot count");
    DBuf vals(dev_, values.size()), work(dev_, evab_encode_work_bytes(dev_->ctx(), 1) / 8);
    dev_->upload(vals.get(), values.data(), values.size() * 8, stream);
    const double *ptr = reinterpret_cast<const double *>(vals.get());
    const std::uint32_t vec = (std::uint32_t)values.size();
    check(evab_encode(dev_->ctx(), 1, &ptr, &vec, &scale, ell, d_pt, work.get(), stream));
    dev_->sync(stream);  // staging buffers are released at scope exit
  }
  // host path (same arithmetic, kept as a cross-check of the device encoder)
  void encodeHost(const std::vector<double> &values, double scale, int ell, u64 *d_pt, void *stream = nullptr) const {
    std::vector<u64> coef;
    embed(values, scale, ell, coef);
    dev_->upload(d_pt, coef.data(), coef.size() * 8, stream);
    std::vector<int> idx(ell);
    for (int i = 0; i < ell; i++) idx[i] = i;
    check(evab_ntt_fwd(dev_->ctx(), d_pt, (std::size_t)ell, idx.data(), ell, stream));
    dev_->sync(stream);
  }
  // decode device plaintext d_pt[ell][N] (NTT form) -> N/2 real slot values: inverse NTT, CRT composition and the FP64
  // forward FFT all run on the device (evab_decode); only the N/2 doubles come back.  (ell > 8: host composition, unembed.)
  std::vector<double> decode(const u64 *d_pt, int ell, double scale) const {
    if (ell <= 8) {
      DBuf out(dev_, N_ / 2), work(dev_, evab_decode_work_bytes(dev_->ctx(), ell) / 8 + 1);
      check(evab_decode(dev_->ctx(), ell, d_pt, scale, reinterpret_cast<double *>(out.get()), work.get(), nullptr));
      std::vector<double> v(N_ / 2);
      dev_->download(v.data(), out.get(), v.size() * 8);
      dev_->sync();
      return v;
    }
    DBuf tmp(dev_, (std::size_t)ell * N_);
    check(evab_add_plain(dev_->ctx(), ell, tmp.get(), d_pt, 1, zeroPlain(ell), nullptr));
    std::vector<int> idx(ell);
    for (int i = 0; i < ell; i++) idx[i] = i;
    check(evab_ntt_inv(dev_->ctx(), tmp.get(), (std::size_t)ell, idx.data(), ell, nullptr));
    std::vector<u64> coef((std::size_t)ell * N_);
    dev_->download(coef.data(), tmp.get(), coef.size() * 8);
    dev_->sync();
    return unembed(coef, ell, scale);
  }
  std::vector<double> unembed(const std::vector<u64> &coef, int ell, double scale) const {
    const auto &P = dev_->primes();
    const int nw = ell + 1;
    std::vector<u64> Q(nw, 0), halfQ(nw);
    Q[0] = 1;
    for (int i = 0; i < ell; i++) bigMul(Q, P[i]);
    std::vector<std::vector<u64>> punct(ell, std::vector<u64>(nw, 0));
    std::vector<u64> ipunct(ell);
    for (int i = 0; i < ell; i++) {
      punct[i][0] = 1;
      for (int j = 0; j < ell; j++) if (j != i) bigMul(punct[i], P[j]);
      ipunct[i] = hmod::inv(bigMod(punct[i], P[i]), P[i]);
    }
    halfQ = Q;  // (Q+1)/2
    { u64 carry = 1; for (int i = 0; i < nw && carry; i++) { halfQ[i] += carry; carry = halfQ[i] == 0; } }
    for (int i = 0; i < nw; i++) halfQ[i] = (halfQ[i] >> 1) | (i + 1 < nw ? halfQ[i + 1] << 63 : 0);
    std::vector<double> re(N_), im(N_, 0.0);
    const double invScale = 1.0 / scale, two64 = 18446744073709551616.0;
    std::vector<u64> X(nw), T(nw);
    for (u64 j = 0; j < N_; j++) {
      std::fill(X.begin(), X.end(), 0);
      for (int i = 0; i < ell; i++) bigAddMul(X, punct[i], hmod::mul(coef[(std::size_t)i * N_ + j], ipunct[i], P[i]));
      while (bigCmp(X, Q) >= 0) bigSub(X, Q);
      const bool neg = bigCmp(X, halfQ) >= 0;
      if (neg) { T = Q; bigSub(T, X); X = T; }
      double acc = 0.0, f = invScale;
      for (int i = 0; i < nw; i++) { if (X[i]) acc += (double)X[i] * f; f *= two64; }
      re[j] = neg ? -acc : acc;
    }
    u64 t = N_;
    for (u64 m = 1; m < N_; m <<= 1) {  // forward special FFT (Cooley-Tukey)
      t >>= 1;
      for (u64 i = 0; i < m; i++) {
        const double wr = rootRe_[m + i], wi = rootIm_[m + i];
        const u64 base = 2 * i * t;
        for (u64 j = base; j < base + t; j++) {
          const double vr = re[j + t] * wr - im[j + t] * wi, vi = re[j + t] * wi + im[j + t] * wr;
          const double ur = re[j], ui = im[j];
          re[j] = ur + vr; im[j] = ui + vi; re[j + t] = ur - vr; im[j + t] = ui - vi;
        }
      }
    }
    std::vector<double> out(N_ / 2);
    for (u64 i = 0; i < N_ / 2; i++) out[i] = re[slotIndex_[i]];
    return out;
  }
  // lazily created all-zero plaintext on the device (used as a copy helper)
  const u64 *zeroPlain(int ell) const {
    std::lock_guard<std::mutex> g(mu_);
    if (!zero_ || zero_.words() < (std::size_t)ell * N_) {
      zero_ = DBuf(dev_, (std::size_t)dev_->k() * N_);
      std::vector<u64> z((std::size_t)dev_->k() * N_, 0);
      dev_->upload(zero_.get(), z.data(), z.size() * 8);
      dev_->sync();
    }
    return zero_.get();
  }

private:
  u64 bitrev(u64 x) const { u64 r = 0; for (int i = 0; i < logN_; i++) { r = (r << 1) | (x & 1); x >>= 1; } return r; }
  // e^(2 pi i index / degree) from the first octant + symmetries
  static void unitRoot(u64 index, u64 degree, double &re, double &im) {
    const double PI = 3.1415926535897932384626433832795028842;
    index &= degree - 1;
    double a, b;
    if (index <= degree / 8) { const double ang = 2.0 * PI * (double)index / (double)degree; re = std::cos(ang); im = std::sin(ang); }
    else if (index <= degree / 4) { unitRoot(degree / 4 - index, degree, a, b); re = b; im = a; }
    else if (index <= degree / 2) { unitRoot(degree / 2 - index, degree, a, b); re = -a; im = b; }
    else if (index <= 3 * degree / 4) { unitRoot(index - degree / 2, degree, a, b); re = -a; im = -b; }
    else { unitRoot(degree - index, degree, a, b); re = a; im = -b; }
  }
  typedef unsigned __int128 u128;
  static void bigMul(std::vector<u64> &a, u64 m) { u64 c = 0; for (auto &w : a) { u128 t = (u128)w * m + c; w = (u64)t; c = (u64)(t >> 64); } }
  static void bigAddMul(std::vector<u64> &acc, const std::vector<u64> &a, u64 m) {
    u64 c = 0;
    for (std::size_t i = 0; i < acc.size(); i++) { u128 t = (u128)a[i] * m + acc[i] + c; acc[i] = (u64)t; c = (u64)(t >> 64); }
  }
  static int bigCmp(const std::vector<u64> &a, const std::vector<u64> &b) {
    for (int i = (int)a.size() - 1; i >= 0; i--) if (a[i] != b[i]) return a[i] > b[i] ? 1 : -1;
    return 0;
  }
  static void bigSub(std::vector<u64> &a, const std::vector<u64> &b) {
    u64 br = 0;
    for (std::size_t i = 0; i < a.size(); i++) { u128 t = (u128)a[i] - b[i] - br; a[i] = (u64)t; br = (u64)(t >> 64) & 1; }
  }
  static u64 bigMod(const std::vector<u64> &a, u64 p) { u64 r = 0; for (int i = (int)a.size() - 1; i >= 0; i--) r = (u64)((((u128)r << 64) | a[i]) % p); return r; }

  std::shared_ptr<Device> dev_;
  u64 N_;
  int logN_;
  std::vector<double> rootRe_, rootIm_;
  std::vector<std::uint32_t> slotIndex_;
  mutable std::mutex mu_;
  mutable DBuf zero_;
};

// the 32-byte seed from which a key-switch key's c1 rows are expanded (key_expand.cuh)
using KeySeed = std::array<std::uint8_t, 32>;

// c1 rows of the keys at d_keys [n][k-1][2][k][N] from the seeds at d_seeds [n][32] (device), modulo the context's primes
inline void expandKeys(Device &dev, int n, const u64 *d_seeds, u64 *d_keys, void *stream) {
  check(evab_expand_key_uniform(dev.ctx(), n, reinterpret_cast<const std::uint8_t *>(d_seeds), dev.primes().data(), d_keys, stream));
}

// the c1 rows of n seed-compressed ciphertexts: entry i writes ell[i] rows at the device pointer c1[i] from seeds[i], modulo the
// context's primes (key_expand.cuh, ciphertext rows); stream-ordered
inline void expandCiphers(Device &dev, int n, const KeySeed *seeds, u64 *const *c1, const int *ell, void *stream) {
  check(evab_expand_cipher_uniform(dev.ctx(), n, reinterpret_cast<const std::uint8_t *>(seeds), c1, ell, dev.primes().data(), stream));
}

// a full key-switch key on the device from its compressed form: host c0 rows [k-1][k][N] and the seed
inline DBuf expandCompressedKey(const std::shared_ptr<Device> &dev, const u64 *c0, const KeySeed &seed) {
  const std::size_t kN = (std::size_t)dev->k() * dev->N();
  DBuf key(dev, (std::size_t)(dev->k() - 1) * 2 * kN), d_seed(dev, 4);
  check(evab_upload_2d(dev->ctx(), key.get(), 2 * kN * 8, c0, kN * 8, kN * 8, (std::size_t)dev->k() - 1, nullptr));
  dev->upload(d_seed.get(), seed.data(), 32);
  expandKeys(*dev, 1, d_seed.get(), key.get(), nullptr);
  dev->sync();
  return key;
}

// Secret / public / evaluation keys resident on the device.
struct KeySet {
  DBuf sk;                       // [k][N]
  DBuf pk;                       // [2][k][N]
  DBuf relin;                    // [k-1][2][k][N]
  std::map<u64, DBuf> galois;    // galois element -> [k-1][2][k][N]
  // seeds of the evaluation keys whose c1 rows are expanded from one (keys from generate_keys, or loaded compressed); keys
  // supplied in full have none
  std::optional<KeySeed> relinSeed;
  std::map<u64, KeySeed> galoisSeeds;
};

class CkksClient {
public:
  // seed == 0: ChaCha20 stream keyed with 256 bits of OS entropy (the secure default); any other value: a deterministic
  // stream for reproducible tests and fixtures ONLY (csprng.hpp)
  CkksClient(std::shared_ptr<Device> dev, std::uint64_t seed) : dev_(std::move(dev)), enc_(dev_), rng_(seed), N_(dev_->N()), k_(dev_->k()) {}
  CkksEncoder &encoder() { return enc_; }

  void keygen(KeySet &K, const std::vector<int> &rotationSteps) {
    std::vector<int> s(N_);
    for (auto &v : s) v = (int)rng_.below(3) - 1;  // uniform ternary
    K.sk = smallToDeviceNtt(s, k_);
    K.pk = DBuf(dev_, (std::size_t)2 * k_ * N_);
    encZeroSym(K, K.pk.get(), K.pk.get() + (std::size_t)k_ * N_);
    DBuf s2(dev_, (std::size_t)k_ * N_);
    check(evab_mul_plain(dev_->ctx(), k_, s2.get(), K.sk.get(), 1, K.sk.get(), nullptr));
    // every evaluation key: a fresh seed from the stream (its c1 rows are expanded on the device), then its digits' errors
    K.relinSeed = drawSeed();
    K.relin = makeKswitchKey(K, s2.get(), *K.relinSeed);
    for (int step : rotationSteps) {
      const u64 elt = evab_galois_elt_from_step(N_, step);
      if (!elt) throw std::invalid_argument("step count too large");
      if (K.galois.count(elt)) continue;
      check(evab_galois_prepare(dev_->ctx(), elt));
      // rotated secret key: one "polynomial" of k residues through the rotate-free permutation path
      DBuf rot(dev_, (std::size_t)k_ * N_);
      permute(rot.get(), K.sk.get(), elt);
      const KeySeed seed = drawSeed();
      K.galoisSeeds[elt] = seed;
      K.galois.emplace(elt, makeKswitchKey(K, rot.get(), seed));
    }
    dev_->sync();
  }
  // Encryptor::encrypt with the public key; d_pt[ell][N]; returns ct [2][ell][N]
  DBuf encrypt(const KeySet &K, const u64 *d_pt, int ell) {
    std::vector<int> u(N_);
    for (auto &v : u) v = (int)rng_.below(3) - 1;
    const std::vector<int> e0 = sampleCbd(), e1 = sampleCbd();
    return encryptWith(K, d_pt, ell, u, e0, e1);
  }
  // the deterministic core (also a test hook: the same (u, e0, e1) through the oracle gives the same bits):
  // (pk0 u + e0, pk1 u + e1) one level up, divided by the extra prime with rounding, + the plaintext
  DBuf encryptWith(const KeySet &K, const u64 *d_pt, int ell, const std::vector<int> &u, const std::vector<int> &e0, const std::vector<int> &e1) {
    if (ell < 1 || ell > k_ - 1) throw std::invalid_argument("encryption level out of range");
    if (u.size() != N_ || e0.size() != N_ || e1.size() != N_) throw std::invalid_argument("randomness must have N entries");
    const int nres = ell + 1;
    DBuf ud = smallToDeviceNtt(u, nres);
    DBuf big(dev_, (std::size_t)2 * nres * N_);
    for (int c = 0; c < 2; c++) {
      DBuf e = smallToDeviceNtt(c ? e1 : e0, nres);
      u64 *dst = big.get() + (std::size_t)c * nres * N_;
      check(evab_mul_plain(dev_->ctx(), nres, dst, K.pk.get() + (std::size_t)c * k_ * N_, 1, ud.get(), nullptr));
      check(evab_add_plain(dev_->ctx(), nres, dst, dst, 1, e.get(), nullptr));
    }
    DBuf ct(dev_, (std::size_t)2 * ell * N_);
    DBuf work(dev_, evab_rescale_work_bytes(dev_->ctx(), 2) / 8);
    check(evab_rescale(dev_->ctx(), nres, ct.get(), big.get(), 2, work.get(), nullptr));
    check(evab_add_plain(dev_->ctx(), ell, ct.get(), ct.get(), 2, d_pt, nullptr));
    dev_->sync();
    return ct;
  }
  // Encryptor::encrypt_symmetric with a seed-compressed result; d_pt[ell][N].  Draws, in this order: a fresh 32-byte seed (4 words of
  // the client's stream), then the error e (sampleCbd, N words).  Returns ct [2][ell][N] and the seed; only c0 (the first ell N
  // words) has to travel, c1 is the seed's expansion
  std::pair<DBuf, KeySeed> encryptSeeded(const KeySet &K, const u64 *d_pt, int ell) {
    const KeySeed seed = drawSeed();
    const std::vector<int> e = sampleCbd();
    return {encryptSeededWith(K, d_pt, ell, seed, e), seed};
  }
  // the deterministic core (also a test hook): c1 = a expanded from `seed` on the device, c0 = -(a s + e) + pt on the first ell
  // residues of s.  No special-prime lift: the encryption is made at its level, as SEAL's symmetric path does
  DBuf encryptSeededWith(const KeySet &K, const u64 *d_pt, int ell, const KeySeed &seed, const std::vector<int> &e) {
    if (!K.sk) throw std::runtime_error("secret-key encryption needs the secret key: this context has none");
    if (ell < 1 || ell > k_ - 1) throw std::invalid_argument("encryption level out of range");
    if (e.size() != N_) throw std::invalid_argument("the error must have N entries");
    const std::size_t P = (std::size_t)ell * N_;
    DBuf ct(dev_, 2 * P);
    u64 *c0 = ct.get(), *c1 = ct.get() + P;
    expandCiphers(*dev_, 1, &seed, &c1, &ell, nullptr);
    DBuf ed = smallToDeviceNtt(e, ell);
    check(evab_mul_plain(dev_->ctx(), ell, c0, c1, 1, K.sk.get(), nullptr));
    check(evab_add_plain(dev_->ctx(), ell, c0, c0, 1, ed.get(), nullptr));
    check(evab_negate(dev_->ctx(), ell, c0, c0, 1, nullptr));
    check(evab_add_plain(dev_->ctx(), ell, c0, c0, 1, d_pt, nullptr));
    dev_->sync();
    return ct;
  }
  // Decryptor::decrypt: pt = c0 + c1 s + c2 s^2; returns device plaintext [ell][N]
  DBuf decrypt(const KeySet &K, const u64 *d_ct, int size, int ell) {
    const std::size_t P = (std::size_t)ell * N_;
    DBuf pt(dev_, P), t(dev_, P), sp(dev_, P);
    check(evab_add_plain(dev_->ctx(), ell, pt.get(), d_ct, 1, enc_.zeroPlain(ell), nullptr));
    check(evab_add_plain(dev_->ctx(), ell, sp.get(), K.sk.get(), 1, enc_.zeroPlain(ell), nullptr));
    for (int i = 1; i < size; i++) {
      check(evab_mul_plain(dev_->ctx(), ell, t.get(), d_ct + (std::size_t)i * P, 1, sp.get(), nullptr));
      check(evab_add_plain(dev_->ctx(), ell, pt.get(), pt.get(), 1, t.get(), nullptr));
      if (i + 1 < size) check(evab_mul_plain(dev_->ctx(), ell, sp.get(), sp.get(), 1, K.sk.get(), nullptr));
    }
    dev_->sync();
    return pt;
  }

private:
  std::vector<int> sampleCbd() {  // centred binomial, 21 - 21 bits (sigma ~ 3.2)
    std::vector<int> e(N_);
    for (auto &v : e) { const u64 x = rng_(); v = __builtin_popcountll(x & 0x1FFFFF) - __builtin_popcountll((x >> 21) & 0x1FFFFF); }
    return e;
  }
  DBuf smallToDeviceNtt(const std::vector<int> &v, int nres) {
    const auto &P = dev_->primes();
    std::vector<u64> r((std::size_t)nres * N_);
    for (int i = 0; i < nres; i++)
      for (u64 j = 0; j < N_; j++) r[(std::size_t)i * N_ + j] = v[j] >= 0 ? (u64)v[j] : P[i] - (u64)(-v[j]);
    DBuf d(dev_, r.size());
    dev_->upload(d.get(), r.data(), r.size() * 8);
    std::vector<int> idx(nres);
    for (int i = 0; i < nres; i++) idx[i] = i;
    check(evab_ntt_fwd(dev_->ctx(), d.get(), (std::size_t)nres, idx.data(), nres, nullptr));
    dev_->sync();
    return d;
  }
  DBuf uniformDevice() {
    const auto &P = dev_->primes();
    std::vector<u64> r((std::size_t)k_ * N_);
    for (int i = 0; i < k_; i++) {
      const u64 p = P[i], lim = UINT64_MAX - (UINT64_MAX % p) - 1;
      for (u64 j = 0; j < N_; j++) { u64 v; do { v = rng_(); } while (v > lim); r[(std::size_t)i * N_ + j] = v % p; }
    }
    DBuf d(dev_, r.size());
    dev_->upload(d.get(), r.data(), r.size() * 8);
    dev_->sync();
    return d;
  }
  KeySeed drawSeed() {
    KeySeed s;
    for (int i = 0; i < 4; i++) {
      const u64 v = rng_();
      for (int b = 0; b < 8; b++) s[8 * i + b] = (std::uint8_t)(v >> (8 * b));
    }
    return s;
  }
  // (c0, c1) = (-(a s + e), a) at key level, NTT form
  void encZeroSym(const KeySet &K, u64 *c0, u64 *c1) {
    DBuf a = uniformDevice();
    check(evab_add_plain(dev_->ctx(), k_, c1, a.get(), 1, enc_.zeroPlain(k_), nullptr));
    maskWith(K, c1, c0);
  }
  // c0 = -(a s + e) for the uniform a at d_a, with a fresh error e
  void maskWith(const KeySet &K, const u64 *d_a, u64 *c0) {
    DBuf e = smallToDeviceNtt(sampleCbd(), k_);
    check(evab_mul_plain(dev_->ctx(), k_, c0, d_a, 1, K.sk.get(), nullptr));
    check(evab_add_plain(dev_->ctx(), k_, c0, c0, 1, e.get(), nullptr));
    check(evab_negate(dev_->ctx(), k_, c0, c0, 1, nullptr));
    dev_->sync();
  }
  // key[J] = (-(a_J s + e_J) + P * newKey on residue J, a_J), the a_J expanded from `seed` on the device
  DBuf makeKswitchKey(const KeySet &K, const u64 *d_newKey, const KeySeed &seed) {
    const auto &P = dev_->primes();
    DBuf key(dev_, (std::size_t)(k_ - 1) * 2 * k_ * N_), d_seed(dev_, 4);
    dev_->upload(d_seed.get(), seed.data(), 32);
    expandKeys(*dev_, 1, d_seed.get(), key.get(), nullptr);
    DBuf t(dev_, (std::size_t)k_ * N_), f(dev_, (std::size_t)k_ * N_);
    std::vector<u64> fh((std::size_t)k_ * N_);
    for (int J = 0; J < k_ - 1; J++) {
      u64 *c0 = key.get() + ((std::size_t)J * 2 + 0) * k_ * N_, *c1 = key.get() + ((std::size_t)J * 2 + 1) * k_ * N_;
      maskWith(K, c1, c0);
      std::fill(fh.begin(), fh.end(), 0);
      const u64 fac = P[k_ - 1] % P[J];
      for (u64 j = 0; j < N_; j++) fh[(std::size_t)J * N_ + j] = fac;
      dev_->upload(f.get(), fh.data(), fh.size() * 8);
      check(evab_mul_plain(dev_->ctx(), k_, t.get(), d_newKey, 1, f.get(), nullptr));
      check(evab_add_plain(dev_->ctx(), k_, c0, c0, 1, t.get(), nullptr));
      dev_->sync();
    }
    return key;
  }
  // out[k][N] = NTT-domain automorphism of in[k][N] (no key switching): done on the
  // host via the same table formula the device uses (setup-time only)
  void permute(u64 *d_out, const u64 *d_in, u64 elt) {
    int logN = 0;
    while ((u64(1) << logN) < N_) logN++;
    auto br = [&](u64 x) { u64 r = 0; for (int i = 0; i < logN; i++) { r = (r << 1) | (x & 1); x >>= 1; } return r; };
    std::vector<u64> in((std::size_t)k_ * N_), out((std::size_t)k_ * N_);
    dev_->download(in.data(), d_in, in.size() * 8);
    dev_->sync();
    for (u64 i = 0; i < N_; i++) {
      const u64 src = br(((elt * (2 * br(i) + 1)) >> 1) & (N_ - 1));
      for (int r = 0; r < k_; r++) out[(std::size_t)r * N_ + i] = in[(std::size_t)r * N_ + src];
    }
    dev_->upload(d_out, out.data(), out.size() * 8);
    dev_->sync();
  }

  std::shared_ptr<Device> dev_;
  CkksEncoder enc_;
  ChaChaRng rng_;
  u64 N_;
  int k_;
};

}  // namespace evab
