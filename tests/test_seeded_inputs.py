"""Seed-compressed input ciphertexts, on the CPU: the ciphertext rows of the expansion rule (row id 2^62 | m, DESIGN §2) replayed
from eva_b200/csrc/key_expand.cuh against an independent numpy implementation, and their separation from key rows."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as o
from test_compressed_keys import HIGH_REJECTION, candidates, np_chacha, np_expand, replay, seeds_for

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
u64p = C.POINTER(C.c_uint64)
CIPHER_ROW = 1 << 62
SENTINEL = 0xDEADBEEF

_LIB = None


def cipher_emu():
    """tests/emu/emu_cipher_expand.cpp, built on first use (like the other emulator libraries)"""
    global _LIB
    if _LIB is None:
        src = os.path.join(ROOT, "tests", "emu", "emu_cipher_expand.cpp")
        so = os.path.join(ROOT, "tests", "emu", "libevab_emu_cipher_expand.so")
        deps = [src, os.path.join(ROOT, "eva_b200", "csrc", "key_expand.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            tmp = "%s.%d" % (so, os.getpid())      # concurrent test workers: each builds its own file, the rename is atomic
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", src, "-o", tmp])
            os.replace(tmp, so)
        lib = C.CDLL(so)
        lib.emu_expand_cipher_uniform.argtypes = [C.c_uint32, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, u64p]
        _LIB = lib
    return _LIB


def np_row(seed, N, q, r):
    """row id r of the rule from its 32-byte seed, modulo q: (the N coefficients, how many took the fallback).  Key rows are
    r = J k + m, ciphertext rows r = 2^62 | m"""
    key = np.frombuffer(seed, dtype="<u4")
    lim = np.uint64(q * ((2 ** 64 - 1) // q))
    cand = candidates(np_chacha(key, np.arange(N // 8), r)).reshape(N)
    row = cand % np.uint64(q)
    todo = np.nonzero(cand >= lim)[0]
    fell = todo.size
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
    return row, fell


def np_cipher_c1(seed, N, moduli, ell):
    """c1 [ell][N] of a seeded ciphertext, and the fallback count of every row"""
    rows = [np_row(seed, N, int(moduli[m]), CIPHER_ROW | m) for m in range(ell)]
    return np.stack([r for r, _ in rows]), np.array([f for _, f in rows])


def replay_cipher(seeds, ells, N, moduli):
    """emulator: one ciphertext [2][ell_i][N] per entry, c0 left at a sentinel, c1 expanded; returns the c1 halves"""
    lib = cipher_emu()
    cts = [np.full((2, ell, N), SENTINEL, dtype=np.uint64) for ell in ells]
    ptrs = np.array([ct.ctypes.data + ell * N * 8 for ct, ell in zip(cts, ells)], dtype=np.uint64)
    sd = np.frombuffer(b"".join(seeds), dtype=np.uint8).copy()
    el = np.array(ells, dtype=np.int32)
    qa = np.array(moduli, dtype=np.uint64)
    assert lib.emu_expand_cipher_uniform(N, len(seeds), sd.ctypes.data, ptrs.ctypes.data, el.ctypes.data, qa.ctypes.data_as(u64p)) == 0
    for ct in cts:
        assert (ct[0] == SENTINEL).all()      # c0 untouched
    return [ct[1] for ct in cts]


def test_row_function_is_the_key_rule_on_key_rows():
    """np_row generalises the key rule's numpy reference: on key rows r = J k + m it gives np_expand's rows"""
    N = 1024
    moduli = o.gen_primes(N, [60] * 3)
    for sd in seeds_for(2, 3):
        want, fell = np_expand(sd, N, moduli)
        for r in range(6):
            J, m = divmod(r, 3)
            row, f = np_row(sd, N, int(moduli[m]), r)
            assert np.array_equal(row, want[J, m]) and f == fell[r]
    # and on high-rejection moduli, where the fallback is taken
    sd = seeds_for(1, 4)[0]
    want, fell = np_expand(sd, N, HIGH_REJECTION)
    row, f = np_row(sd, N, HIGH_REJECTION[1], 4)
    assert np.array_equal(row, want[1, 1]) and f == fell[4] > 0


def test_cipher_replay_equals_numpy_on_a_seal_chain():
    N = 16384
    moduli = o.gen_primes(N, [60, 40, 40, 40, 60])
    seeds = seeds_for(4, 16384)
    ells = [1, 2, 3, 4]
    got = replay_cipher(seeds, ells, N, moduli)
    for sd, ell, c1 in zip(seeds, ells, got):
        want, _ = np_cipher_c1(sd, N, moduli, ell)
        assert np.array_equal(c1, want), ell
        assert (c1 < np.array(moduli[:ell], dtype=np.uint64)[:, None]).all()
    # a lower level is the prefix of a higher one: row m depends on (seed, m) only
    same = replay_cipher([seeds[0]] * 2, [1, 4], N, moduli)
    assert np.array_equal(same[0], same[1][:1])


@pytest.mark.parametrize("N", [1024, 4096])
def test_cipher_replay_equals_numpy_with_high_rejection_moduli(N):
    """every row takes the fallback, and the replay still equals the numpy reference word for word"""
    seeds = seeds_for(2, 91 + N)
    got = replay_cipher(seeds, [3, 2], N, HIGH_REJECTION)
    for sd, ell, c1 in zip(seeds, [3, 2], got):
        want, fell = np_cipher_c1(sd, N, HIGH_REJECTION, ell)
        assert (fell > 0).all(), fell
        assert np.array_equal(c1, want)


def test_cipher_rows_and_key_rows_under_one_seed_differ():
    """nonce domain separation: a ciphertext and a key expanded from the same seed share no row and no 60-bit value"""
    N = 4096
    moduli = o.gen_primes(N, [60] * 5)
    sd = seeds_for(1, 17)[0]
    key_c1 = replay([sd], N, moduli)[0, :, 1]           # [k-1][k][N]
    ct_c1 = replay_cipher([sd], [4], N, moduli)[0]      # [4][N]
    for m in range(4):
        for J in range(4):
            assert not np.array_equal(ct_c1[m], key_c1[J, m])
    assert np.intersect1d(ct_c1.ravel(), key_c1.ravel()).size == 0
    assert np.unique(ct_c1).size == ct_c1.size
    # two seeds give different ciphertext rows; the same seed the same rows
    other = replay_cipher(seeds_for(2, 17)[1:], [4], N, moduli)[0]
    assert not any(np.array_equal(other[m], ct_c1[m]) for m in range(4))
    assert np.array_equal(replay_cipher([sd], [4], N, moduli)[0], ct_c1)
