"""Compact responses, on the CPU: the compaction element of evab_compact_ciphers and the client elements of evab_compact_unpack /
evab_compact_finish (eva_b200/csrc/compact_kernels.cuh, replayed by tests/emu/emu_compact.cpp) against the definition computed with
Python integers; the packed layout against numpy; the width rule; and the checks of the compact value kind and of the option."""
import ctypes as C
import math
import os
import random
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
u64p = C.POINTER(C.c_uint64)

_LIB = None


def emu():
    """tests/emu/emu_compact.cpp, built on first use (like the other emulator libraries)"""
    global _LIB
    if _LIB is None:
        src = os.path.join(ROOT, "tests", "emu", "emu_compact.cpp")
        so = os.path.join(ROOT, "tests", "emu", "libevab_emu_compact.so")
        deps = [src] + [os.path.join(ROOT, "eva_b200", "csrc", f) for f in ("compact_kernels.cuh", "encode_kernels.cuh", "modarith.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            tmp = "%s.%d" % (so, os.getpid())      # concurrent test workers: each builds its own file, the rename is atomic
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", src, "-o", tmp])
            os.replace(tmp, so)
        lib = C.CDLL(so)
        lib.emu_compact.argtypes = [C.c_uint32, C.c_int, u64p, C.c_int, C.c_int, u64p, u64p]
        lib.emu_compact_unpack.argtypes = [C.c_uint32, C.c_int, u64p, C.c_int, u64p, u64p]
        lib.emu_compact_finish.argtypes = [C.c_uint32, C.c_int, u64p, C.c_int, u64p, C.c_int, u64p, C.c_void_p]
        _LIB = lib
    return _LIB


def _p(a):
    return a.ctypes.data_as(u64p)


def is_prime(n):
    if n < 2:
        return False
    for p in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        if n % p == 0:
            return n == p
    d, s = n - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for a in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        x = pow(a, d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def ntt_primes(bits, N, count):
    """the `count` largest primes below 2^bits that are 1 mod 2N (the shape of the context's primes)"""
    out, q = [], (2 ** bits // (2 * N)) * 2 * N + 1
    while len(out) < count:
        q -= 2 * N
        if is_prime(q):
            out.append(q)
    return out


PRIMES = {(bits, N): ntt_primes(bits, N, 8) for bits in (60, 30) for N in (1024, 16384)}


# ------------------------------------------------------------------------------------------------ the definition, Python integers
def crt(residues, primes):
    Q = math.prod(primes)
    x = 0
    for r, q in zip(residues, primes):
        m = Q // q
        x += int(r) * m * pow(m, -1, q)
    return x % Q


def compact_ref(xs, Q, shift, bits):
    """y = floor((2^(shift+1) x + Q) / (2Q)) mod 2^bits of every coefficient"""
    return [((x << (shift + 1)) + Q) // (2 * Q) % (1 << bits) for x in xs]


def pack_ref(ys, bits):
    """numpy bit packing: field i at bits [i bits, (i+1) bits) of a little-endian stream, zero-padded to whole u64 words"""
    y = np.array(ys, dtype=np.uint64)
    bitmat = ((y[:, None] >> np.arange(bits, dtype=np.uint64)[None, :]) & np.uint64(1)).astype(np.uint8).reshape(-1)
    W = (len(ys) * bits + 63) // 64
    bitmat = np.concatenate([bitmat, np.zeros(W * 64 - bitmat.size, dtype=np.uint8)])
    return np.packbits(bitmat, bitorder="little").view("<u8").astype(np.uint64)


def residues_of(xs, primes):
    return np.array([[x % q for x in xs] for q in primes], dtype=np.uint64)


def boundary_values(Q, shift, rng, count):
    """x = 0, Q - 1 and the neighbours of rounding boundaries (k + 1/2) Q / 2^shift"""
    xs = [0, Q - 1, 1, Q // 2, Q // 2 + 1]
    while len(xs) < count:
        k = rng.randrange(1 << min(shift, 4096))
        x0 = (2 * k + 1) * Q >> (shift + 1)
        xs += [v for v in (x0 - 1, x0, x0 + 1) if 0 <= v < Q]
    return xs[:count]


def run_compact(N, primes, shift, bits, xs0, xs1):
    ell = len(primes)
    coef = np.ascontiguousarray(np.stack([residues_of(xs0, primes), residues_of(xs1, primes)]))
    W = (N * bits + 63) // 64
    dst = np.full((2, W), 0xA5A5A5A5A5A5A5A5, dtype=np.uint64)
    qa = np.array(primes, dtype=np.uint64)
    assert emu().emu_compact(N, ell, _p(qa), shift, bits, _p(coef), _p(dst)) == 0
    return dst


def check_compact(N, primes, shift, bits, rng, live=None):
    """live: only the first and last `live` coefficients are non-zero (x = 0 gives y = 0), which keeps the big-integer reference
    cheap at N = 16384 while the head and the tail words of the stream are exercised"""
    Q = math.prod(primes)
    n = N if live is None else 2 * live
    xs0 = boundary_values(Q, shift, rng, n // 2) + [rng.randrange(Q) for _ in range(n - n // 2)]
    xs1 = [rng.randrange(Q) for _ in range(n)]
    if live is not None:
        xs0 = xs0[:live] + [0] * (N - n) + xs0[live:]
        xs1 = xs1[:live] + [0] * (N - n) + xs1[live:]
    got = run_compact(N, primes, shift, bits, xs0, xs1)
    want = np.stack([pack_ref(compact_ref(xs0, Q, shift, bits), bits), pack_ref(compact_ref(xs1, Q, shift, bits), bits)])
    assert np.array_equal(got, want), (N, len(primes), primes[0].bit_length(), shift, bits)


@pytest.mark.parametrize("qbits", [60, 30])
@pytest.mark.parametrize("ell", range(1, 9))
def test_compaction_equals_the_definition_n1024(qbits, ell):
    """every width 1..62 and shift in {b, b+1, b+17}; ell = 1 takes the 128-by-64 division, ell > 1 the multi-word one"""
    N = 1024
    primes = PRIMES[(qbits, N)][:ell]
    rng = random.Random(1000 * qbits + ell)
    for bits in range(1, 63):
        for shift in (bits, bits + 1, bits + 17):
            check_compact(N, primes, shift, bits, rng)


@pytest.mark.parametrize("qbits", [60, 30])
@pytest.mark.parametrize("ell", [1, 2, 5, 8])
def test_compaction_equals_the_definition_n16384(qbits, ell):
    """every width 1..62 and shift in {b, b+1, b+17} at N = 16384: the last word of every width that does not divide 64"""
    N = 16384
    primes = PRIMES[(qbits, N)][:ell]
    rng = random.Random(7 * qbits + ell)
    for bits in range(1, 63):
        for shift in (bits, bits + 1, bits + 17):
            check_compact(N, primes, shift, bits, rng, live=256)
    check_compact(N, primes, 60, 37, rng)         # one fully random polynomial pair


def test_compaction_of_a_full_shift_and_large_shift():
    """shift far above every prime (the headroom of a large-range output dropped) and the Sobel shape itself"""
    rng = random.Random(3)
    primes = PRIMES[(60, 16384)][:1]
    check_compact(16384, primes, 60, 37, rng)
    check_compact(1024, PRIMES[(30, 1024)][:3], 200, 40, rng)


@pytest.mark.parametrize("bits", [1, 3, 7, 13, 31, 32, 33, 37, 47, 57, 61, 62])
def test_unpack_reads_the_packed_layout(bits):
    """evab_compact_unpack's element: field i of the numpy-packed stream, modulo every prime (fields can exceed a 30-bit prime)"""
    N = 1024
    rng = np.random.default_rng(bits)
    ys = [int(v) for v in rng.integers(0, 1 << bits, size=2 * N, dtype=np.uint64)]
    words = np.ascontiguousarray(np.stack([pack_ref(ys[:N], bits), pack_ref(ys[N:], bits)]))
    for primes in (PRIMES[(60, N)][:2], PRIMES[(30, N)][:3]):
        qa = np.array(primes, dtype=np.uint64)
        out = np.zeros((2, len(primes), N), dtype=np.uint64)
        assert emu().emu_compact_unpack(N, len(primes), _p(qa), bits, _p(words), _p(out)) == 0
        want = np.stack([residues_of(ys[:N], primes), residues_of(ys[N:], primes)])
        assert np.array_equal(out, want)


@pytest.mark.parametrize("bits", [1, 2, 17, 37, 62])
def test_finish_centres_mod_2b_and_rewrites_residues(bits):
    """evab_compact_finish's element: the CRT value v of y0 + y1 s in (-P/2, P/2] -> z = v mod 2^b centred to (-2^(b-1), 2^(b-1)]"""
    N = 1024
    rng = random.Random(bits)
    for primes, nout in ((PRIMES[(60, N)][:2], 2), (PRIMES[(30, N)][:4], 3)):
        P = math.prod(primes)
        vs = [rng.randrange(-(P // 2), P // 2 + 1) for _ in range(N - 4)] + [0, 1, -1, P // 2]
        coef = residues_of([v % P for v in vs], primes)
        qa = np.array(primes, dtype=np.uint64)
        out = np.zeros((nout, N), dtype=np.uint64)
        z = np.zeros(N, dtype=np.int64)
        assert emu().emu_compact_finish(N, len(primes), _p(qa), bits, _p(coef), nout, _p(out), z.ctypes.data) == 0
        half = 1 << (bits - 1)
        wz = [(v % (1 << bits)) - (1 << bits) if v % (1 << bits) > half else v % (1 << bits) for v in vs]
        assert z.tolist() == wz
        assert np.array_equal(out, residues_of([v % math.prod(primes[:nout]) for v in wz], primes[:nout]))


def test_client_path_inverts_the_compaction():
    """compaction of a fresh symmetric encryption of m, then the client's arithmetic in Python integers: z = Delta' m + small noise"""
    N, bits, p = 1024, 40, 8
    primes = PRIMES[(60, N)][:2]
    Q = math.prod(primes)
    rng = random.Random(9)
    s = [rng.choice((-1, 0, 1)) for _ in range(N)]
    a = [rng.randrange(Q) for _ in range(N)]
    m = [rng.randrange(-(1 << 30), 1 << 30) for _ in range(N)]
    as_ = negacyclic(a, s)
    c0 = [(m[i] + rng.randrange(-8, 9) - as_[i]) % Q for i in range(N)]
    shift = math.ceil(math.log2(Q)) + p
    words = run_compact(N, primes, shift, bits, c0, a)
    y0 = fields(words[0], bits, N)
    y1 = fields(words[1], bits, N)
    ys = negacyclic(y1, s)
    z = [(y0[i] + ys[i]) % (1 << bits) for i in range(N)]
    z = [v - (1 << bits) if v > 1 << (bits - 1) else v for v in z]
    ratio = 2.0 ** shift / Q
    assert max(abs(z[i] - m[i] * ratio) for i in range(N)) < 8 * ratio + N   # encryption error times the ratio, rounding noise


def negacyclic(a, s):
    N = len(a)
    out = [0] * N
    for j, sj in enumerate(s):
        if sj:
            for i in range(N):
                k = i + j
                if k < N:
                    out[k] += sj * a[i]
                else:
                    out[k - N] -= sj * a[i]
    return out


def fields(words, bits, N):
    v = int.from_bytes(np.asarray(words, dtype="<u8").tobytes(), "little")
    return [(v >> (i * bits)) & ((1 << bits) - 1) for i in range(N)]


# ------------------------------------------------------------------------------------------------ the width rule
def shape_ref(primes, ell, scale, rng_bits, p, N):
    log2Q = 0.0
    for q in primes[:ell]:
        log2Q += math.log2(float(q))
    m = int(math.log2(N)) + 1
    shift = math.ceil(log2Q - math.log2(scale)) + p + m
    bits = min(shift, rng_bits + p + m + 2)
    return bits < math.floor(log2Q) and bits <= 62, shift, bits, 2.0 ** (math.log2(scale) + shift - log2Q)


def _module():
    from eva_b200 import _eva_b200 as m
    return m


@pytest.mark.parametrize("N,prime_bits,scale_bits,range_bits,p,bits,response", [
    (16384, [60], 25, 10, 10, 37, 151552),    # Sobel
    (16384, [60], 25, 10, 20, 47, 192512),
    (16384, [60], 25, 20, 10, 47, 192512),    # Harris
    (16384, [60], 25, 20, 20, 57, 233472),
])
def test_width_rule_table(N, prime_bits, scale_bits, range_bits, p, bits, response):
    m = _module()
    primes = m._b200.create_coeff_modulus(N, prime_bits)
    compact, shift, b, scale = m._compact_shape(primes, 1, 2.0 ** scale_bits, range_bits, p, N)
    assert compact and b == bits and 2 * ((N * b + 63) // 64) * 8 == response
    assert (compact, shift, b, scale) == shape_ref(primes, 1, 2.0 ** scale_bits, range_bits, p, N)
    assert 2.0 ** (shift - 60) < scale / 2.0 ** scale_bits < 2.0 ** (shift - 59)


def test_width_rule_polynomial_and_full_cases():
    m = _module()
    N = 8192
    primes = m._b200.create_coeff_modulus(N, [60, 60])
    # b = shift: no headroom to drop (range 30 at scale 2^30 in a 60-bit prime), and compaction still shrinks at p = 10
    compact, shift, b, _ = m._compact_shape(primes, 1, 2.0 ** 30, 30, 10, N)
    assert compact and b == shift == 54
    # p = 20: b = 64 > 62, stays full
    compact, shift, b, _ = m._compact_shape(primes, 1, 2.0 ** 30, 30, 20, N)
    assert not compact and b == 64
    # b >= floor(log2 Q): nothing would shrink
    compact, _, b, _ = m._compact_shape(primes, 1, 2.0 ** 20, 40, 6, N)
    assert not compact and b == 60
    # two output primes: ell 64-bit words shrink to b bits
    compact, _, b, _ = m._compact_shape(primes, 2, 2.0 ** 40, 20, 10, N)
    assert compact and b == 20 + 10 + 14 + 2
    for ell, scale, rb, p in ((1, 2.0 ** 25, 10, 1), (2, 2.0 ** 50, 5, 52), (1, 2.0 ** 59, 0, 3), (2, 2.0 ** 30, 60, 8)):
        assert m._compact_shape(primes, ell, scale, rb, p, N) == shape_ref(primes, ell, scale, rb, p, N)


def test_width_rule_stays_full_for_the_other_cases():
    """size 3, not a ciphertext, no declared range, more than 8 residues: full, whatever the width would be"""
    m = _module()
    N = 8192
    primes = m._b200.create_coeff_modulus(N, [60, 60])
    assert m._compact_shape(primes, 1, 2.0 ** 30, 30, 10, N)[0]
    assert not m._compact_shape(primes, 1, 2.0 ** 30, 30, 10, N, size=3)[0]
    assert not m._compact_shape(primes, 1, 2.0 ** 30, 30, 10, N, cipher=False)[0]
    assert not m._compact_shape(primes, 1, 2.0 ** 30, None, 10, N)[0]
    primes9 = m._b200.create_coeff_modulus(N, [30] * 10)
    compact, _, b, _ = m._compact_shape(primes9, 8, 2.0 ** 30, 10, 10, N)
    assert compact and b == 36
    compact, _, b, _ = m._compact_shape(primes9, 9, 2.0 ** 30, 10, 10, N)
    assert not compact and b == 36


# ------------------------------------------------------------------------------------------------ the value kind
@pytest.mark.parametrize("shape,bits", [((2, 10), 0), ((2, 10), 63), ((3, 592), 37), ((2,), 37), ((2, 593), 37), ((1, 592), 37)])
def test_bad_compact_values_raise(shape, bits):
    from eva_b200 import b200
    val = b200.B200Valuation()
    with pytest.raises((ValueError, RuntimeError)):
        val.set_compact_cipher("out", np.zeros(shape, dtype=np.uint64), bits, 1.0)
    with pytest.raises((ValueError, RuntimeError, IndexError, KeyError)):
        val.compact_bits("out")


def test_set_options_refuses_out_of_range_precision():
    from eva_b200 import _eva_b200 as m
    opt = m._PlanOptions()
    for bad in (-1, 53, 100):
        with pytest.raises(ValueError, match="compact_outputs"):
            opt.set_options(compact_outputs=bad)
    opt.set_options(compact_outputs=52)
