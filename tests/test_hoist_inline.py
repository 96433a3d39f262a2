"""Inline hoist constants (evab_set_hoist_inline, B200Server(hoist_constants="inline")) replayed on the CPU: the hoisted rotations
that form each constant from the key rows they load and the element's indicator rows equal, word for word, the same rotations
reading the stored constants -- from a key bank of two tenants with different keys, at every level, on chains where q_J mod m is
and is not trivial -- and the oracle's rotate_vector."""
import ctypes as C

import numpy as np
import pytest

import parity_cases as pc
from backends import _elt, _p
from oracle import oracle as o
from test_rotation_wsum import WSUM_STEPS, WSUM_VALUES, WsumEmuBackend
from test_tenants import Bank


class InlineEmu(WsumEmuBackend):
    """the emulator with the inline replays (tests/emu/emu_inline.cpp: emui_*) beside the key-bank ones (emub_*)"""
    SRC, LIB = "emu_inline.cpp", "libevab_emu_inline"

    def __init__(self, N, primes):
        super().__init__(N, primes)
        for fn in ("emu_hoist_indicators_bytes", "emu_rotate_modup_many_work_bytes"):
            getattr(self.lib, fn).restype = C.c_size_t

    def indicators(self, elts):
        out = np.empty((len(elts), self.k, self.N), dtype=np.uint64)
        assert self.lib.emu_hoist_indicators_bytes(self.h, len(elts)) == out.nbytes
        self._chk(self.lib.emu_hoist_indicators(self.h, len(elts), (C.c_uint64 * len(elts))(*elts), _p(out)))
        return out


class InlineBank:
    """the keys-only layout of an inline key bank (relinearization key, then one Galois key per sorted element) and the one shared
    copy of the elements' indicator rows [n][k][N]"""

    def __init__(self, be, orcs, elts):
        N, k = be.N, be.k
        self.elts, self.kw = elts, (k - 1) * 2 * k * N
        self.stride = self.kw * (1 + len(elts))
        self.words = np.zeros((len(orcs), self.stride), dtype=np.uint64)
        for t, orc in enumerate(orcs):
            self.words[t, :self.kw] = orc.relin_key().ravel()
            for i, e in enumerate(elts):
                self.words[t, self.kw * (1 + i):self.kw * (2 + i)] = orc.galois_key(e).ravel()
        self.ind = be.indicators(elts)

    def key(self, e):
        return self.words.ctypes.data + 8 * self.kw * (1 + self.elts.index(e))

    def ind_ptr(self, e):
        return self.ind[self.elts.index(e)].ctypes.data


def _ptrs(xs):
    return (C.c_void_p * max(1, len(xs)))(*xs)


class Case:
    """one chain, two tenants with different keys, both banks; run(t, fn) selects tenant t's region in the instance table"""

    def __init__(self, N, bits, steps):
        self.orcs = [o.Oracle(N, bits).keygen(seed) for seed in (21, 22)]
        self.be = InlineEmu(N, self.orcs[0].primes)
        self.N, self.k = N, self.be.k
        self.steps = list(steps)
        self.bank = Bank(self.be, self.orcs, self.steps)
        self.ibank = InlineBank(self.be, self.orcs, self.bank.elts)
        self.table = np.zeros(1, dtype=np.int32)
        self.lib = self.be.lib

    def select(self, t, stride):
        self.table[0] = t
        self.lib.emu_set_key_bank(self.table.ctypes.data_as(C.c_void_p), C.c_size_t(stride))

    def prepare(self, a, scale_c0):
        ell = a.shape[1]
        that, ext, z = np.empty((ell, self.N), dtype=np.uint64), np.zeros((ell + 1, ell, self.N), dtype=np.uint64), np.zeros(1, dtype=np.uint64)
        self.be._chk(self.lib.emu_rotate_modup_prepare(self.be.h, ell, _p(that), _p(ext), _p(a), _p(z)))
        if scale_c0:
            self.be._chk(self.lib.emu_rotate_modup_scale_c0(self.be.h, ell, _p(ext), _p(a)))
        assert z[0] == 0
        return ext

    def stored(self, elts, ell):
        return [self.bank.ptr(self.bank.galois_off(e)) for e in elts], [self.bank.ptr(self.bank.cadd_off(e, ell)) for e in elts]

    def inline(self, elts):
        return [self.ibank.key(e) for e in elts], [self.ibank.ind_ptr(e) for e in elts]

    def both(self, t, call):
        """call(prefix, keys, cadds) under tenant t of the stored bank and of the inline bank"""
        try:
            self.select(t, self.bank.stride)
            want = call("emub_", *self.stored_args)
            self.select(t, self.ibank.stride)
            got = call("emui_", *self.inline_args)
        finally:
            self.lib.emu_set_key_bank(None, C.c_size_t(0))
        return got, want

    def args(self, steps, ell):
        elts = [_elt(self.N, s) for s in steps]
        self.stored_args, self.inline_args = self.stored(elts, ell), self.inline(elts)
        return elts

    # ---- the three C-ABI ops
    def modup_prepared(self, t, a, step):
        ell = a.shape[1]
        ext = self.prepare(a, scale_c0=False)
        elt, = self.args([step], ell)

        def call(pre, keys, cadds):
            out = np.empty((2, ell, self.N), dtype=np.uint64)
            work = np.zeros(self.lib.emu_rotate_modup_work_bytes(self.be.h, ell) // 8, dtype=np.uint64)
            self.be._chk(getattr(self.lib, pre + "rotate_modup_prepared")(self.be.h, ell, _p(out), _p(a), _p(ext), C.c_uint64(elt),
                                                                           C.c_void_p(keys[0]), C.c_void_p(cadds[0]), _p(work)))
            return out
        return self.both(t, call)

    def modup_many(self, t, a, steps):
        ell, n = a.shape[1], len(steps)
        ext = self.prepare(a, scale_c0=True)
        elts = self.args(steps, ell)

        def call(pre, keys, cadds):
            out = np.empty((n, 2, ell, self.N), dtype=np.uint64)
            work = np.zeros(self.lib.emu_rotate_modup_many_work_bytes(self.be.h, ell, n) // 8, dtype=np.uint64)
            self.be._chk(getattr(self.lib, pre + "rotate_modup_many")(self.be.h, ell, n, _p(out), _p(a), _p(ext), (C.c_uint64 * n)(*elts),
                                                                       _ptrs(keys), _ptrs(cadds), _p(work)))
            return out
        return self.both(t, call)

    def wsum(self, t, a, steps, nout, seed):
        orc, ell, n = self.orcs[t], a.shape[1], len(steps)
        ext = self.prepare(a, scale_c0=True)
        elts = self.args(steps, ell)
        rng = np.random.default_rng(seed)
        enc = lambda v: orc.encode(np.array([v]), 2.0 ** 30, ell)
        wts = [[None if rng.random() < 0.2 else enc(WSUM_VALUES[rng.integers(len(WSUM_VALUES))]) for _ in range(n)] for _ in range(nout)]
        y = pc.rand_ct(orc, 2, ell, 700 + seed)
        taps = [a, y]
        twts = [[enc(-1.0 - oi), None if oi % 2 else enc(0.25 * oi + 0.5)] for oi in range(nout)]
        ptr = lambda w: None if w is None else w.ctypes.data

        def call(pre, keys, cadds):
            out = np.empty((nout, 2, ell, self.N), dtype=np.uint64)
            work = np.zeros(self.lib.emu_rotate_wsum_work_bytes(self.be.h, ell, n, nout) // 8, dtype=np.uint64)
            self.be._chk(getattr(self.lib, pre + "rotate_wsum")(self.be.h, ell, nout, _p(out), _p(a), _p(ext), n, (C.c_uint64 * n)(*elts),
                                                                 _ptrs(keys), _ptrs(cadds), _ptrs([ptr(w) for ws in wts for w in ws]), len(taps),
                                                                 _ptrs([x.ctypes.data for x in taps]), _ptrs([ptr(w) for ws in twts for w in ws]),
                                                                 _p(work)))
            return out
        got, want = self.both(t, call)
        return got, want, (wts, taps, twts)


CHAINS = {
    "60bit": (1024, [60, 60, 60, 60]),
    "mixed60_50": (1024, [60, 50, 50, 60]),          # q_J mod m is a real reduction for every pair of different sizes
    "k6": (1024, [60, 50, 60, 50, 50, 60]),
}
STEPS = WSUM_STEPS        # 16 distinct elements


@pytest.fixture(scope="module", params=sorted(CHAINS))
def case(request):
    return Case(*CHAINS[request.param], STEPS)


def test_indicator_rows_are_the_stored_constants_factor(case):
    """ind[g][m] equals NTT_m(I_g), the factor the stored constants were built with: cadd_g[c][m] = ind[row(m)] (.) sum_J (q_J mod m)
    K_g[J][c][m] -- restated in numpy from the keys, for every element, level and tenant"""
    N, k, primes = case.N, case.k, case.orcs[0].primes
    for gi, e in enumerate(case.bank.elts[:4]):
        ind = case.ibank.ind[gi]
        for t in (0, 1):
            K = case.orcs[t].galois_key(e)
            for ell in range(1, k):
                stored = case.bank.words[t, case.bank.cadd_off(e, ell):case.bank.cadd_off(e, ell) + 2 * (ell + 1) * N].reshape(2, ell + 1, N)
                for mi in range(ell + 1):
                    row = mi if mi < ell else k - 1
                    p = int(primes[row])
                    for c in range(2):
                        s = sum(int(primes[J]) % p * K[J, c, row].astype(object) for J in range(ell)) % p
                        want = (s * ind[row].astype(object)) % p
                        assert np.array_equal(stored[c, mi], want.astype(np.uint64)), (e, t, ell, mi, c)


@pytest.mark.parametrize("t", [0, 1])
def test_rotate_modup_prepared_inline_equals_stored(case, t):
    orc = case.orcs[t]
    for ell in range(1, case.k):
        a = pc.rand_ct(orc, 2, ell, 100 * ell + t)
        for s in STEPS[:3]:
            got, want = case.modup_prepared(t, a, s)
            pc.eq(got, want)
    # the oracle's rotate_vector with tenant t's own key
    ell = case.k - 1
    a = pc.rand_ct(orc, 2, ell, 55 + t)
    got, _ = case.modup_prepared(t, a, 7)
    pc.eq(got, orc.rotate(a, 7, orc.galois_key(o.galois_elt_from_step(case.N, 7))))


@pytest.mark.parametrize("t", [0, 1])
@pytest.mark.parametrize("n", [1, 3, 16])
def test_rotate_modup_many_inline_equals_stored(case, t, n):
    orc = case.orcs[t]
    for ell in range(1, case.k):
        a = pc.rand_ct(orc, 2, ell, 300 + 10 * ell + n + t)
        got, want = case.modup_many(t, a, STEPS[:n])
        pc.eq(got, want)
        if ell == case.k - 1 and n == 3:
            for i, s in enumerate(STEPS[:n]):
                pc.eq(got[i], orc.rotate(a, s, orc.galois_key(o.galois_elt_from_step(case.N, s))))


@pytest.mark.parametrize("t", [0, 1])
@pytest.mark.parametrize("nout", [1, 2, 3, 4])
def test_rotate_wsum_inline_equals_stored(case, t, nout):
    orc = case.orcs[t]
    for ell in range(1, case.k):
        n = (5, 16, 8, 3)[ell % 4]
        a = pc.rand_ct(orc, 2, ell, 500 + 10 * ell + nout + t)
        got, want, (wts, taps, twts) = case.wsum(t, a, STEPS[:n], nout, seed=ell * 7 + nout)
        pc.eq(got, want)
        if ell == case.k - 1:   # rotate -> multiply_plain -> add in the oracle, with tenant t's keys
            rots = [orc.rotate(a, s, orc.galois_key(o.galois_elt_from_step(case.N, s))) for s in STEPS[:n]]
            for oi in range(nout):
                acc = None
                for c_, w in list(zip(rots, wts[oi])) + list(zip(taps, twts[oi])):
                    if w is not None:
                        term = orc.mul_plain(c_, w)
                        acc = term if acc is None else orc.add(acc, term)
                pc.eq(got[oi], acc)


def test_tenants_differ_and_indicators_stay_put():
    """two tenants of the same inline bank give different words (their keys differ) and each its own stored result: an indicator
    moved by the tenant offset would read tenant 1's keys as indicator rows"""
    c = Case(*CHAINS["mixed60_50"], STEPS[:4])
    outs = []
    for t in (0, 1):
        a = pc.rand_ct(c.orcs[0], 2, 2, 9)
        got, want = c.modup_many(t, a, STEPS[:4])
        pc.eq(got, want)
        outs.append(got)
    assert not np.array_equal(outs[0], outs[1])


def test_lazy_rotsum_refuses_inline():
    c = Case(*CHAINS["60bit"], STEPS[:2])
    ell = 2
    a = pc.rand_ct(c.orcs[0], 2, ell, 3)
    ext = c.prepare(a, scale_c0=True)
    elts = c.args(STEPS[:2], ell)
    keys, inds = c.inline_args
    c.lib.emu_lazy_rotsum_work_bytes.restype = C.c_size_t
    work = np.zeros(c.lib.emu_lazy_rotsum_work_bytes(c.be.h, ell, 1) // 8, dtype=np.uint64)
    wt = np.zeros((ell + 1, c.N), dtype=np.uint64)
    out = np.empty((1, 2, ell, c.N), dtype=np.uint64)
    rc = c.lib.emui_lazy_rotsum(c.be.h, ell, 1, _p(out), _p(a), _p(ext), 2, (C.c_uint64 * 2)(*elts), _ptrs(keys), _ptrs(inds),
                                _ptrs([wt.ctypes.data, wt.ctypes.data]), _p(work))
    assert rc != 0 and b"approx_hoist" in c.lib.emu_last_error()
