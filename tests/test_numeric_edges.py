"""Numeric edges of the kernels, against the oracle bit for bit:

* the encoder at coefficient magnitudes on both sides of every branch and table boundary of enc_residue (2^64, 2^128, 2^192,
  ..., up to the largest finite doubles), with signs, -0.0 and exact ties, through every encoder entry point;
* every op on 60-bit prime chains at the edge of the two-row fold arithmetic (p = 2^60 - delta, delta just below and just
  above 2^25), with the fold path and the lazy Shoup path forced in turn, and the longest 60-bit chain a 128-bit-secure
  program has at N = 32768 (14 primes of SEAL's scan);
* the same prime-edge matrix on a CPU replay built with -DEVAB_BOUND_CHECK, which checks every compile-time bound of the
  fold arithmetic against the value it describes;
* decoding on the 14-prime chain: the device decoder (ell <= 8) and the host composition (ell > 8).
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import parity_cases as pc
from backends import ROOT, GpuBackend, _p
from oracle import oracle as o
from test_rotation_wsum import WsumEmuBackend, WsumGpuBackend, case_rotation_wsum

FOLD_DELTA = 1 << 25       # modarith.cuh prime_foldable: p = 2^60 - delta with delta < 2^25


def foldmask(primes):
    return sum(1 << i for i, p in enumerate(primes) if (1 << 60) - p < FOLD_DELTA)


def edge_primes(N, count, foldable):
    """60-bit primes p = 1 mod 2N next to the fold threshold: the `count` fold-friendly ones with the largest delta (scanning
    upwards from 2^60 - 2^25 + 1) or the `count` others with the smallest delta (scanning downwards from just below it)"""
    start = (1 << 60) - FOLD_DELTA + 1
    p, step = (start, 2 * N) if foldable else (start - 2 * N, -2 * N)
    out = []
    while len(out) < count:
        if o.lib.ora_is_prime(C.c_uint64(p)):
            out.append(p)
        p += step
    return out


def chains(N):
    """the hand-picked chains (the last prime is the key-switch prime P)"""
    f, n = edge_primes(N, 5, True), edge_primes(N, 5, False)
    return {"fold": f, "nofold": n, "mixed": [n[0], f[0], n[1], f[1], n[2]]}


_ORACLES = {}


def oracle_for(N, primes):
    key = (N, tuple(primes))
    if key not in _ORACLES:
        _ORACLES[key] = o.Oracle(N, primes=list(primes)).keygen(3)
    return _ORACLES[key]


# ---- encoder magnitude sweep -------------------------------------------------------------------------------------------

MANTISSAS = (1.0, 1.7254603006834726, 2.0 - 2.0 ** -52, 1.0 + 2.0 ** -52)


def sweep_scalars(modbits):
    """(value, scale) pairs whose coefficient round(value * scale) sits at 2^m for m on both sides of each boundary of
    enc_residue (the 2^64 branch, the old 2^128-entry table), just under the modulus and far above it (largest exponent
    of a finite double); signs, -0.0, exact ties"""
    out = []
    for m in (52, 63, 64, 65, 127, 128, 191, 192, 255, 256, modbits - 2, modbits + 40, 700, 1000, 1023):
        for f in MANTISSAS:
            for sgn in (1.0, -1.0):
                out.append((sgn * f * 2.0 ** (m - 60), 2.0 ** 60))
        out.append((1.0, 2.0 ** m))                        # the magnitude in the scale alone
    for v in (0.0, -0.0, 0.5, -0.5, 2.5, -2.5, 3.5, 2.0 ** 51 + 0.5, -(2.0 ** 51 + 0.5)):
        out.append((v, 1.0))                               # v * scale = k + 1/2 exactly: rounds away from zero
    out.append((1.25, 2.0))                                # 2.5 after scaling
    return out


def sweep_vectors(N):
    """vectors whose inverse-FFT coefficients spread over the same magnitudes"""
    rng = np.random.default_rng(N + 5)
    out = []
    for a in (3, 62, 126, 134, 190, 200, 260, 400, 900):
        out.append((rng.uniform(-1, 1, N // 2) * 2.0 ** a, 2.0 ** 60))
        out.append((np.array([2.0 ** a, -(2.0 ** a) * 0.75]), 2.0 ** 60))
    out.append((np.array([-0.0, 0.0, 2.5, -2.5]), 1.0))
    return out


def p_row(orc, coef_src_values, scale):
    """the residue row mod the key-switch prime P that encode_ext(with_p=1) appends: the oracle's encoder on a context whose
    first prime is P"""
    P = orc.primes[-1]
    key = (orc.N, P)
    if key not in _ORACLES:
        _ORACLES[key] = o.Oracle(orc.N, primes=[P, orc.primes[0]])
    return _ORACLES[key].encode(coef_src_values, scale, 1)[0]


def emu_encode_ext(be, vecs, scale, ell):
    n = len(vecs)
    vecs = [np.ascontiguousarray(v, dtype=np.float64) for v in vecs]
    out = np.empty((n, ell + 1, be.N), dtype=np.uint64)
    work = np.zeros(be.lib.emu_encode_work_bytes(be.h, n) // 8, dtype=np.uint64)
    be._chk(be.lib.emu_encode_ext(be.h, n, (C.c_void_p * n)(*[v.ctypes.data for v in vecs]), (C.c_uint32 * n)(*[len(v) for v in vecs]),
                                  (C.c_double * n)(*[scale] * n), ell, 1, _p(out), _p(work)))
    return out


def emu_encode_uniform_ext(be, values, scale, ell):
    n = len(values)
    out = np.empty((n, ell + 1, be.N), dtype=np.uint64)
    be._chk(be.lib.emu_encode_uniform_ext(be.h, n, (C.c_double * n)(*values), (C.c_double * n)(*[scale] * n), ell, 1, _p(out)))
    return out


def gpu_encode_ext(be, vecs, scale, ell):
    lib, n = be.lib, len(vecs)
    dv = [be._up(np.ascontiguousarray(v, dtype=np.float64).view(np.uint64)) for v in vecs]
    do = be._alloc(n * (ell + 1) * be.N * 8)
    dw = be._alloc(lib.evab_encode_work_bytes(be.h, n))
    be._chk(lib.evab_encode_ext(be.h, n, (C.c_void_p * n)(*dv), (C.c_uint32 * n)(*[len(v) for v in vecs]), (C.c_double * n)(*[scale] * n),
                                ell, 1, do, dw, None))
    out = be._down(do, (n, ell + 1, be.N))
    be._free(do, dw, *dv)
    return out


def gpu_encode_uniform_ext(be, values, scale, ell):
    n = len(values)
    do = be._alloc(n * (ell + 1) * be.N * 8)
    be._chk(be.lib.evab_encode_uniform_ext(be.h, n, (C.c_double * n)(*values), (C.c_double * n)(*[scale] * n), ell, 1, do, None))
    out = be._down(do, (n, ell + 1, be.N))
    be._free(do)
    return out


def case_encode_sweep(orc, uniform, vector, with_p=None, ells=None):
    """uniform(values, scale, ell) -> [n][ell][N] and vector(vec, scale, ell) -> [ell][N] against Oracle.encode; with_p = (uniform_ext,
    vector_ext) adds the plaintexts with the extra row mod P"""
    ells = ells or (orc.k,)
    modbits = sum(int(p).bit_length() for p in orc.primes[:max(ells)])
    scalars = sweep_scalars(modbits)
    for ell in ells:
        by_scale = {}
        for v, s in scalars:
            by_scale.setdefault(s, []).append(v)
        for s, vals in by_scale.items():
            got = uniform(vals, s, ell)
            for e, v in enumerate(vals):
                pc.eq(got[e], orc.encode(np.array([v]), s, ell))
        for vec, s in sweep_vectors(orc.N):
            pc.eq(vector(vec, s, ell), orc.encode(vec, s, ell))
    if with_p:
        uni_ext, vec_ext = with_p
        ell = orc.k - 1
        for s in (2.0 ** 60, 1.0):
            vals = [v for v, s_ in scalars if s_ == s]
            got = uni_ext(vals, s, ell)
            for e, v in enumerate(vals):
                pc.eq(got[e][:ell], orc.encode(np.array([v]), s, ell))
                pc.eq(got[e][ell], p_row(orc, np.array([v]), s))
        vecs = sweep_vectors(orc.N)
        for s in (2.0 ** 60, 1.0):
            vs = [v for v, s_ in vecs if s_ == s]
            got = vec_ext(vs, s, ell)
            for e, v in enumerate(vs):
                pc.eq(got[e][:ell], orc.encode(v, s, ell))
                pc.eq(got[e][ell], p_row(orc, v, s))


def test_encoder_magnitudes_emulated():
    """enc_residue is exact for every finite coefficient: the CPU replay of the encoder kernels on a 300-bit modulus"""
    N = 1024
    for primes in (o.gen_primes(N, [60] * 5), chains(N)["mixed"]):
        orc = oracle_for(N, primes)
        be = WsumEmuBackend(N, orc.primes)
        case_encode_sweep(orc, be.encode_uniform, lambda v, s, ell: be.encode([v], s, ell)[0],
                          with_p=(lambda vals, s, ell: emu_encode_uniform_ext(be, vals, s, ell), lambda vs, s, ell: emu_encode_ext(be, vs, s, ell)),
                          ells=(orc.k, 2))


@pytest.mark.gpu
@pytest.mark.parametrize("N,chain", [(1024, "seal5"), (1024, "mixed"), (32768, "seal14")])
def test_encoder_magnitudes_gpu(N, chain):
    """the device encoders (evab_encode_uniform, evab_encode, their _ext rows mod P) and the host encoder behind
    B200Public.encode, at every magnitude of the sweep"""
    from eva_b200 import b200
    primes = {"seal5": lambda: o.gen_primes(N, [60] * 5), "seal14": lambda: o.gen_primes(N, [60] * 14), "mixed": lambda: chains(N)["mixed"]}[chain]()
    orc = seal14_oracle() if chain == "seal14" else oracle_for(N, primes)
    be = GpuBackend(N, orc.primes)
    pub = b200.public_from_raw(N, orc.primes, orc.public_key(), None, {})
    ells = (orc.k - 1, 2)
    case_encode_sweep(orc, be.encode_uniform, lambda v, s, ell: pub.encode(list(v), s, ell),
                      with_p=(lambda vals, s, ell: gpu_encode_uniform_ext(be, vals, s, ell), lambda vs, s, ell: gpu_encode_ext(be, vs, s, ell)),
                      ells=ells)
    case_encode_sweep(orc, lambda vals, s, ell: np.stack([pub.encode([v], s, ell, True) for v in vals]),
                      lambda v, s, ell: pub.encode(list(v), s, ell, True), ells=ells)


# ---- prime-edge chains -------------------------------------------------------------------------------------------------

def case_prime_edges(be, orc, ells):
    """every op family of the parity suite on one chain, and one weighted rotation sum"""
    pc.case_ntt(be, orc)
    for ell in ells:
        pc.case_dyadic(be, orc, ell)
        pc.case_sum_terms(be, orc, ell)
        pc.case_sum_products(be, orc, ell)
        pc.case_keyswitch(be, orc, ell)
        if ell >= 2:
            pc.case_rescale(be, orc, ell)
    pc.case_encode_uniform(be, orc)
    pc.case_decode(be, orc)
    case_rotation_wsum(be, orc, max(ells), 4, 2)


def cpu_prime_edge_matrix(bound_check=False):
    """the hand-picked chains at N = 1024 and 4096, with the fold arithmetic (where every prime of a launch allows it) and the
    lazy Shoup arithmetic forced"""
    for N in (1024, 4096):
        for name, primes in chains(N).items():
            orc = oracle_for(N, primes)
            be = WsumEmuBackend(N, orc.primes, bound_check=bound_check)
            assert be.lib.emu_ctx_foldmask(be.h) == foldmask(primes), name
            for arith in (0, 1):
                assert be.lib.emu_ctx_set_ntt_arith(be.h, arith) == 0
                before = be.lib.emu_fold_launches()
                case_prime_edges(be, orc, (1, orc.k - 1))
                folded = be.lib.emu_fold_launches() - before
                if arith == 0 and name == "fold":
                    assert folded > 0, (N, name)
                if arith == 1 or name == "nofold":
                    assert folded == 0, (N, name, arith)


def test_prime_edges_emulated():
    cpu_prime_edge_matrix()


def test_prime_edges_bound_checked():
    """the same matrix on the replay built with -DEVAB_BOUND_CHECK, in a subprocess: a violated bound aborts that process and
    its `bound violated at ...` line becomes this test's failure"""
    tests = os.path.join(ROOT, "tests")
    code = ("import sys; sys.path[:0] = [%r, %r]\nimport test_numeric_edges as t\nt.cpu_prime_edge_matrix(bound_check=True)\n"
            "print('bound-checked matrix passed')" % (ROOT, tests))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0 and "bound-checked matrix passed" in r.stdout, (r.returncode, r.stdout[-2000:], r.stderr[-4000:])


_SEAL14 = {}


def seal14_oracle():
    """N = 32768 with 14 60-bit primes of SEAL's scan: the longest 60-bit chain of a 128-bit-secure program at that N (its
    delta reaches 2^24.6).  Keys are generated once per session."""
    if not _SEAL14:
        _SEAL14["orc"] = o.Oracle(32768, primes=o.gen_primes(32768, [60] * 14)).keygen(3)
    return _SEAL14["orc"]


@pytest.fixture(scope="module")
def seal14():
    return seal14_oracle()


@pytest.mark.gpu
@pytest.mark.parametrize("N", [4096, 32768])
@pytest.mark.parametrize("name", ["fold", "nofold", "mixed"])
def test_prime_edges_gpu(N, name):
    """the hand-picked chains on the device, fold and lazy Shoup arithmetic; evab_ctx_foldmask marks exactly the primes with
    delta < 2^25"""
    primes = chains(N)[name]
    orc = oracle_for(N, primes)
    be = WsumGpuBackend(N, orc.primes)
    assert be.lib.evab_ctx_foldmask(be.h) == foldmask(primes)
    for arith in (0, 1):
        assert be.lib.evab_ctx_set_ntt_arith(be.h, arith) == 0
        case_prime_edges(be, orc, (1, orc.k - 1))


@pytest.mark.gpu
@pytest.mark.parametrize("cluster,arith", [(0, 0), (0, 1), (2, 0), (4, 0)])
def test_seal14_chain_gpu(seal14, cluster, arith):
    """the 14-prime SEAL-scan chain at N = 32768: every prime is fold-friendly; the library's default cluster and clusters of
    2 and 4 CTAs per residue"""
    orc = seal14
    from eva_b200 import cabi
    lib = cabi.load()
    assert lib.evab_set_ntt_cluster(cluster) == 0
    try:
        be = WsumGpuBackend(orc.N, orc.primes)
    finally:
        assert lib.evab_set_ntt_cluster(0) == 0
    assert be.lib.evab_ctx_foldmask(be.h) == foldmask(orc.primes) == (1 << 14) - 1
    assert be.lib.evab_ctx_set_ntt_arith(be.h, arith) == 0
    pc.case_ntt(be, orc)
    for ell in (orc.k - 1, 7):
        pc.case_dyadic(be, orc, ell)
        pc.case_sum_terms(be, orc, ell, nterms=(9,))
        pc.case_sum_products(be, orc, ell, nterms=(7,))
        pc.case_keyswitch(be, orc, ell)
        pc.case_rescale(be, orc, ell)
    pc.case_encode_uniform(be, orc)
    case_rotation_wsum(be, orc, orc.k - 1, 2, 2)


# ---- long-chain decode -------------------------------------------------------------------------------------------------

def edge_coefficients(Q, N, rng):
    """N integers in [0, Q): the centring threshold and its neighbours, 0, 1, Q - 1, every 64-bit word boundary, the rest
    uniform (every word of the CRT composition in use)"""
    half = (Q + 1) // 2
    special = [0, 1, Q - 1, half - 1, half, half + 1, Q - 2]
    for w in range(1, Q.bit_length() // 64 + 1):
        special += [(1 << (64 * w)) - 1, 1 << (64 * w), Q - (1 << (64 * w))]
    vals = [int(x) % Q for x in special]
    while len(vals) < N:
        vals.append(int.from_bytes(rng.bytes(Q.bit_length() // 8 + 8), "little") % Q)
    return vals


def ntt_form(orc, coefs, ell):
    return np.stack([orc.ntt_fwd(np.array([c % orc.primes[i] for c in coefs], dtype=np.uint64), i) for i in range(ell)])


def same_doubles(got, want, what):
    got = np.ascontiguousarray(np.asarray(got, dtype=np.float64)[: len(want)])
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), what


@pytest.mark.gpu
def test_decode_long_chain_gpu(seal14):
    """the 14-prime chain: ell = 6..8 on the device decoder (evab_decode), ell = 9..13 through the host composition of
    CkksEncoder::decode, for encoder plaintexts and raw residues -- identical doubles to Oracle.decode"""
    from eva_b200 import b200
    orc = seal14
    N = orc.N
    be = GpuBackend(N, orc.primes)
    pub = b200.public_from_raw(N, orc.primes, orc.public_key(), None, {})
    sec = b200.secret_from_raw(N, orc.primes, orc.secret_key())
    rng = np.random.default_rng(14)
    for ell in range(6, orc.k):
        Q = 1
        for p in orc.primes[:ell]:
            Q *= p
        pts = [(orc.encode(rng.uniform(-4, 4, N // 2), 2.0 ** 50, ell), 2.0 ** 50),
               (orc.encode(rng.uniform(-1, 1, N // 2) * 2.0 ** 200, 2.0 ** 60, ell), 2.0 ** 60),
               (ntt_form(orc, edge_coefficients(Q, N, rng), ell), 2.0 ** 40)]
        for i, (pt, scale) in enumerate(pts):
            want = orc.decode(pt, scale)
            if ell <= 8:
                same_doubles(be.decode(pt, scale), want, ("evab_decode", ell, i))
            same_doubles(pub.decode(pt, scale), want, ("public decode", ell, i))
            same_doubles(sec.decode(pt, scale), want, ("secret decode", ell, i))
