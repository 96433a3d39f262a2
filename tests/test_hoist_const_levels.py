"""evab_rotate_hoist_const_levels: the hoist constants of every level of n Galois keys in one pass, replayed on the CPU against
evab_rotate_hoist_const (one call per level), word for word, with oracle keys."""
import ctypes as C

import numpy as np
import pytest

from backends import EmuBackend, _p
from oracle import oracle as o


class LevelsEmuBackend(EmuBackend):
    SRC, LIB = "emu_levels.cpp", "libevab_emu_levels"

    def __init__(self, N, primes):
        super().__init__(N, primes)
        for n in ("emu_hoist_const_levels_bytes", "emu_rotate_hoist_const_levels_work_bytes"):
            getattr(self.lib, n).restype = C.c_size_t

    def levels(self, elts, keys):
        """[n][sum_ell 2 (ell+1) N] from keys [n][k-1][2][k][N]"""
        n = len(elts)
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        out = np.zeros((n, self.lib.emu_hoist_const_levels_bytes(self.h) // 8), dtype=np.uint64)
        tmp = np.zeros(self.lib.emu_rotate_hoist_const_levels_work_bytes(self.h, n) // 8, dtype=np.uint64)
        ea = (C.c_uint64 * n)(*elts)
        self._chk(self.lib.emu_rotate_hoist_const_levels(self.h, n, ea, _p(keys), _p(out), _p(tmp)))
        return out

    def one_level(self, elt, key, ell):
        out = np.empty((2, ell + 1, self.N), dtype=np.uint64)
        tmp = np.empty((ell + 1, self.N), dtype=np.uint64)
        self._chk(self.lib.emu_rotate_hoist_const(self.h, ell, C.c_uint64(elt), _p(np.ascontiguousarray(key)), _p(out), _p(tmp)))
        return out


def level_blocks(block, k, N):
    """split one key's constants into {ell: [2][ell+1][N]}"""
    out, off = {}, 0
    for ell in range(1, k):
        w = 2 * (ell + 1) * N
        out[ell] = block[off:off + w].reshape(2, ell + 1, N)
        off += w
    assert off == block.size
    return out


@pytest.mark.parametrize("N,bits", [(1024, [60, 60, 60]), (1024, [60, 40, 40, 60, 60]), (4096, [60, 60, 60]), (4096, [60, 50, 50, 50, 60]),
                                    (1024, [60] * 18)])
def test_levels_equal_one_call_per_level(N, bits):
    """every (element, level) of the one-pass call equals evab_rotate_hoist_const of that level; the 18-prime chain sums 17 terms"""
    orc = o.Oracle(N, bits).keygen(len(bits))
    be = LevelsEmuBackend(N, orc.primes)
    k = orc.k
    steps = (1, -3, 7) if k < 10 else (1, -3)
    elts = [o.galois_elt_from_step(N, s) for s in steps]
    keys = np.stack([orc.galois_key(e) for e in elts])
    got = be.levels(elts, keys)
    assert got.shape == (len(elts), ((k + 1) * k - 2) * N)
    for g, e in enumerate(elts):
        blocks = level_blocks(got[g], k, N)
        for ell in range(1, k):
            want = be.one_level(e, keys[g], ell)
            assert np.array_equal(blocks[ell], want), (N, k, e, ell)
    # one key alone gives the same block as in the batch (no cross-talk between keys)
    assert np.array_equal(be.levels(elts[-1:], keys[-1:])[0], got[-1])


def test_levels_rejects_bad_arguments():
    orc = o.Oracle(1024, [60, 60]).keygen(1)
    be = LevelsEmuBackend(1024, orc.primes)
    with pytest.raises(RuntimeError, match="n must be"):
        be.levels([], np.zeros((0, 1, 2, 2, 1024), dtype=np.uint64))
