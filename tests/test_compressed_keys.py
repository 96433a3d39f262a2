"""Seed-compressed evaluation keys, on the CPU: the ChaCha20 block function shared by the host CSPRNG and the key expansion
(eva_b200/csrc/key_expand.cuh), and the expansion rule replayed from that header against an independent numpy implementation of
the rule written down in DESIGN §2."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
u32p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
M32 = 0xFFFFFFFF

# moduli between 2^62 and 2^64: a candidate is rejected with probability 40 %, 20 % and 15 % (2^64 mod q over 2^64)
HIGH_REJECTION = [int(0.6 * 2 ** 64) | 1, int(0.4 * 2 ** 64) | 1, int(0.85 * 2 ** 64) | 1]

_LIB = None


def emu():
    """tests/emu/emu_expand.cpp, built on first use (like the other emulator libraries)"""
    global _LIB
    if _LIB is None:
        src = os.path.join(ROOT, "tests", "emu", "emu_expand.cpp")
        so = os.path.join(ROOT, "tests", "emu", "libevab_emu_expand.so")
        deps = [src, os.path.join(ROOT, "eva_b200", "csrc", "key_expand.cuh"), os.path.join(ROOT, "eva_b200", "csrc", "host", "csprng.hpp")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", src, "-o", so])
        lib = C.CDLL(so)
        lib.emu_chacha20_block.argtypes = [u32p, C.c_uint64, C.c_uint64, u32p]
        lib.emu_chacha_rng.argtypes = [C.c_uint64, C.c_int, u64p]
        lib.emu_expand_key_uniform.argtypes = [C.c_uint32, C.c_int, C.c_int, C.c_void_p, u64p, u64p]
        _LIB = lib
    return _LIB


# ------------------------------------------------------------------------------------------------- independent numpy reference
def np_chacha(key, counters, nonces):
    """ChaCha20 blocks [B][16] (uint32) for key words [8] and arrays of 64-bit counters / nonces (RFC 8439, 20 rounds)"""
    counters = np.asarray(counters, dtype=np.uint64)
    nonces = np.broadcast_to(np.asarray(nonces, dtype=np.uint64), counters.shape)
    B = counters.size
    s = np.empty((16, B), dtype=np.uint32)
    s[0:4] = np.array([0x61707865, 0x3320646e, 0x79622d32, 0x6b206574], dtype=np.uint32)[:, None]
    s[4:12] = np.asarray(key, dtype=np.uint32)[:, None]
    s[12], s[13] = (counters & M32).astype(np.uint32), (counters >> np.uint64(32)).astype(np.uint32)
    s[14], s[15] = (nonces & M32).astype(np.uint32), (nonces >> np.uint64(32)).astype(np.uint32)
    x = s.copy()

    def rotl(v, n):
        return (v << np.uint32(n)) | (v >> np.uint32(32 - n))

    def qr(a, b, c, d):
        x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 16)
        x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 12)
        x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 8)
        x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 7)

    for _ in range(10):
        qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
        qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
    return (x + s).T.copy()


def candidates(blocks):
    """[B][16] uint32 -> [B][8] uint64: w[2i] | w[2i+1] << 32"""
    b = blocks.astype(np.uint64)
    return b[:, 0::2] | (b[:, 1::2] << np.uint64(32))


def np_expand(seed, N, moduli):
    """the c1 rows [k-1][k][N] of one key from its 32-byte seed, and for every row the number of coefficients that took the
    fallback"""
    key = np.frombuffer(seed, dtype="<u4")
    k = len(moduli)
    out = np.zeros((k - 1, k, N), dtype=np.uint64)
    fell = np.zeros((k - 1) * k, dtype=int)
    for r in range((k - 1) * k):
        J, m = divmod(r, k)
        q = int(moduli[m])
        lim = np.uint64(q * ((2 ** 64 - 1) // q))
        cand = candidates(np_chacha(key, np.arange(N // 8), r)).reshape(N)
        row = cand % np.uint64(q)
        todo = np.nonzero(cand >= lim)[0]
        fell[r] = todo.size
        t = 0
        while todo.size:
            assert t < 256
            c = candidates(np_chacha(key, todo.astype(np.uint64) * np.uint64(256) + np.uint64(t), (1 << 63) | r))
            ok = c < lim
            first = np.argmax(ok, axis=1)
            done = ok.any(axis=1)
            row[todo[done]] = c[done, first[done]] % np.uint64(q)
            todo = todo[~done]
            t += 1
        out[J, m] = row
    return out, fell


def replay(seeds, N, moduli):
    """emulator: [n][k-1][2][k][N] with only the c1 rows written (the c0 rows keep a marker)"""
    k, n = len(moduli), len(seeds)
    keys = np.full((n, k - 1, 2, k, N), 0xDEADBEEF, dtype=np.uint64)
    sd = np.frombuffer(b"".join(seeds), dtype=np.uint8).copy()
    qa = np.array(moduli, dtype=np.uint64)
    assert emu().emu_expand_key_uniform(N, k, n, sd.ctypes.data, qa.ctypes.data_as(u64p), keys.ctypes.data_as(u64p)) == 0
    assert (keys[:, :, 0] == 0xDEADBEEF).all()       # c0 untouched
    return keys


def seeds_for(n, salt):
    rng = np.random.default_rng(salt)
    return [rng.integers(0, 256, 32, dtype=np.uint8).tobytes() for _ in range(n)]


# ------------------------------------------------------------------------------------------------------------------- tests
RFC8439_KEY = np.frombuffer(bytes(range(32)), dtype="<u4").copy()
# RFC 8439 §2.3.2: block count 1, nonce 00:00:00:09:00:00:00:4a:00:00:00:00 -> state words 12..15 = 1, 0x09000000, 0x4a000000, 0
RFC8439_COUNTER, RFC8439_NONCE = 1 | (0x09000000 << 32), 0x4a000000
RFC8439_OUT = [0xe4e7f110, 0x15593bd1, 0x1fdd0f50, 0xc47120a3, 0xc7f4d1c7, 0x0368c033, 0x9aaa2204, 0x4e6cd4c3,
               0x466482d2, 0x09aa9f07, 0x05d7c214, 0xa2028bd9, 0xd19c12b5, 0xb94e16de, 0xe883d0cb, 0x4e3c50a2]


def test_block_function_rfc8439_vector():
    out = np.zeros(16, dtype=np.uint32)
    emu().emu_chacha20_block(RFC8439_KEY.ctypes.data_as(u32p), RFC8439_COUNTER, RFC8439_NONCE, out.ctypes.data_as(u32p))
    assert [int(v) for v in out] == RFC8439_OUT
    assert [int(v) for v in np_chacha(RFC8439_KEY, [RFC8439_COUNTER], RFC8439_NONCE)[0]] == RFC8439_OUT


def test_host_csprng_is_the_shared_block_function():
    """ChaChaRng(seed) streams the blocks (counter 0, 1, ..; nonce 0) of its SplitMix64-derived key through the shared block"""
    seed = 7
    key, x = [], seed
    for _ in range(4):
        x = (x + 0x9E3779B97F4A7C15) & (2 ** 64 - 1)
        z = x
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & (2 ** 64 - 1)
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & (2 ** 64 - 1)
        z ^= z >> 31
        key += [z & M32, z >> 32]
    want = candidates(np_chacha(np.array(key, dtype=np.uint32), np.arange(3), 0)).reshape(-1)
    got = np.zeros(24, dtype=np.uint64)
    emu().emu_chacha_rng(seed, 24, got.ctypes.data_as(u64p))
    assert np.array_equal(got, want)


@pytest.mark.parametrize("N,nprimes", [(1024, 3), (1024, 5), (4096, 3), (4096, 5)])
def test_replay_equals_numpy_on_seal_chains(N, nprimes):
    moduli = o.gen_primes(N, [60] * nprimes)
    seeds = seeds_for(2, N + nprimes)
    keys = replay(seeds, N, moduli)
    for g, sd in enumerate(seeds):
        want, _ = np_expand(sd, N, moduli)
        assert np.array_equal(keys[g, :, 1], want), (N, nprimes, g)


@pytest.mark.parametrize("N", [1024, 4096])
def test_replay_equals_numpy_with_high_rejection_moduli(N):
    """moduli between 2^62 and 2^64: every row takes the fallback, and the replay still equals the numpy reference word for word"""
    seeds = seeds_for(2, 77 + N)
    keys = replay(seeds, N, HIGH_REJECTION)
    for g, sd in enumerate(seeds):
        want, fell = np_expand(sd, N, HIGH_REJECTION)
        assert (fell > 0).all(), fell
        assert np.array_equal(keys[g, :, 1], want), (N, g)
        assert (keys[g, :, 1] < np.array(HIGH_REJECTION, dtype=np.uint64)[None, :, None]).all()


def test_values_in_range_seeds_differ_rows_do_not_collide():
    N = 4096
    moduli = o.gen_primes(N, [60] * 5)
    a, b = seeds_for(2, 5)
    keys = replay([a, b], N, moduli)
    c1 = keys[:, :, 1]
    assert (c1 < np.array(moduli, dtype=np.uint64)[None, None, :, None]).all()
    # two seeds: no row in common
    assert not any(np.array_equal(c1[0, J, m], c1[1, J, m]) for J in range(4) for m in range(5))
    # the 20 rows of one key draw from 20 distinct nonces: no candidate repeats across rows (60-bit values, 81920 of them)
    for g in range(2):
        assert np.unique(c1[g]).size == c1[g].size
    # the same seed gives the same key
    assert np.array_equal(replay([a], N, moduli)[0], keys[0])
