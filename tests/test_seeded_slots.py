"""Seeded key slots (evab_set_key_seeded, B200Server(key_storage="seeded")) replayed on the CPU: the key switches that draw every
key's c1 words from its seed (tests/emu/emu_seeded.cpp, the SEED bodies and the shared draw of key_expand.cuh) equal, word for word,
the same ops on the expanded keys -- relinearize, rotate, the hoisted single rotation, rotate_modup_many and rotate_wsum at every
level, on a two-tenant bank -- and the oracle's key switch with those keys; the drawn words are np_expand's; the calls that read
expanded keys refuse seeded ones."""
import ctypes as C

import numpy as np
import pytest

import parity_cases as pc
from backends import _elt, _p
from oracle import oracle as o
from test_compressed_keys import HIGH_REJECTION, np_expand, seeds_for
from test_hoist_inline import InlineEmu
from test_rotation_wsum import WSUM_STEPS, WSUM_VALUES


class SeededEmu(InlineEmu):
    """the emulator with the seeded replays (emus_*) beside the inline (emui_*) and key-bank (emub_*) ones"""
    SRC, LIB = "emu_seeded.cpp", "libevab_emu_seeded"

    def __init__(self, N, primes):
        super().__init__(N, primes)
        for fn in ("emus_seeded_key_words", "emu_rotate_modup_work_bytes", "emu_rotate_wsum_work_bytes", "emu_keyswitch_work_bytes",
                   "emu_lazy_rotsum_work_bytes", "emu_rotate_hoist_const_levels_work_bytes", "emu_hoist_const_levels_bytes"):
            if hasattr(self.lib, fn):
                getattr(self.lib, fn).restype = C.c_size_t


def _ptrs(xs):
    return (C.c_void_p * max(1, len(xs)))(*xs)


class Banks:
    """two tenants' keys in the keys-only layout of an expanded inline bank and in the seeded layout (every key an image: c0 rows,
    then the seed padded to 64 bytes).  Each key's c0 rows are the oracle key's, its c1 rows np_expand of a seed: the seeded image
    then stands for exactly that expanded key"""

    def __init__(self, be, orcs, elts, salt):
        N, k = be.N, be.k
        self.elts, self.kw = elts, (k - 1) * 2 * k * N
        self.sw = int(be.lib.emus_seeded_key_words(k, C.c_size_t(N)))
        assert self.sw == (k - 1) * k * N + 8
        nk = 1 + len(elts)
        self.exp = np.zeros((len(orcs), self.kw * nk), dtype=np.uint64)
        self.seeded = np.zeros((len(orcs), self.sw * nk), dtype=np.uint64)
        self.full = []   # [tenant][key index] the expanded keys [k-1][2][k][N]
        seeds = seeds_for(len(orcs) * nk, salt)
        for t, orc in enumerate(orcs):
            keys = [orc.relin_key()] + [orc.galois_key(e) for e in elts]
            full = []
            for i, K in enumerate(keys):
                sd = seeds[t * nk + i]
                c1, _ = np_expand(sd, N, orc.primes)
                F = K.copy()
                F[:, 1] = c1
                full.append(F)
                self.exp[t, self.kw * i:self.kw * (i + 1)] = F.ravel()
                self.seeded[t, self.sw * i:self.sw * i + self.sw - 8] = F[:, 0].ravel()
                self.seeded[t, self.sw * i + self.sw - 8:self.sw * i + self.sw - 4] = np.frombuffer(sd, dtype=np.uint64)
            self.full.append(full)
        self.ind = be.indicators(elts)

    def index(self, e):
        return 0 if e is None else 1 + self.elts.index(e)

    def exp_key(self, e):
        return self.exp.ctypes.data + 8 * self.kw * self.index(e)

    def seeded_key(self, e):
        return self.seeded.ctypes.data + 8 * self.sw * self.index(e)

    def ind_ptr(self, e):
        return self.ind[self.elts.index(e)].ctypes.data


class Case:
    def __init__(self, N, bits, steps, salt=0):
        self.orcs = [o.Oracle(N, bits).keygen(seed) for seed in (31, 32)]
        self.be = SeededEmu(N, self.orcs[0].primes)
        self.N, self.k, self.lib = N, self.be.k, self.be.lib
        self.steps = list(steps)
        self.elts = sorted({_elt(N, s) for s in self.steps})
        self.banks = Banks(self.be, self.orcs, self.elts, salt + N + len(bits))
        self.table = np.zeros(1, dtype=np.int32)

    def select(self, t, stride):
        self.table[0] = t
        self.lib.emu_set_key_bank(self.table.ctypes.data_as(C.c_void_p), C.c_size_t(stride))

    def both(self, t, call, exp_prefix="emui_"):
        """call(prefix, key_of, ind_of) under tenant t of the expanded bank and of the seeded bank"""
        b = self.banks
        try:
            self.select(t, b.exp.shape[1])
            want = call(exp_prefix, b.exp_key, b.ind_ptr)
            self.select(t, b.seeded.shape[1])
            got = call("emus_", b.seeded_key, b.ind_ptr)
        finally:
            self.lib.emu_set_key_bank(None, C.c_size_t(0))
        return got, want

    def key(self, t, e=None):
        return self.banks.full[t][self.banks.index(e)]

    def prepare(self, a, scale_c0):
        ell = a.shape[1]
        that, ext, z = np.empty((ell, self.N), dtype=np.uint64), np.zeros((ell + 1, ell, self.N), dtype=np.uint64), np.zeros(1, dtype=np.uint64)
        self.be._chk(self.lib.emu_rotate_modup_prepare(self.be.h, ell, _p(that), _p(ext), _p(a), _p(z)))
        if scale_c0:
            self.be._chk(self.lib.emu_rotate_modup_scale_c0(self.be.h, ell, _p(ext), _p(a)))
        assert z[0] == 0
        return ext

    def relinearize(self, t, a):
        ell = a.shape[1]

        def call(pre, key, ind):
            out = np.empty((2, ell, self.N), dtype=np.uint64)
            work = np.zeros(self.lib.emu_keyswitch_work_bytes(self.be.h, ell) // 8 + 8 * self.N * (ell + 2), dtype=np.uint64)
            self.be._chk(getattr(self.lib, pre + "relinearize")(self.be.h, ell, _p(out), _p(a), C.c_void_p(key(None)), _p(work)))
            return out
        return self.both(t, call, "emub_")

    def rotate(self, t, a, step):
        ell, elt = a.shape[1], _elt(self.N, step)

        def call(pre, key, ind):
            out = np.empty((2, ell, self.N), dtype=np.uint64)
            work = np.zeros(self.lib.emu_keyswitch_work_bytes(self.be.h, ell) // 8 + 8 * self.N * (ell + 2), dtype=np.uint64)
            self.be._chk(getattr(self.lib, pre + "rotate")(self.be.h, ell, _p(out), _p(a), C.c_uint64(elt), C.c_void_p(key(elt)), _p(work)))
            return out
        return self.both(t, call, "emub_")

    def modup_prepared(self, t, a, step):
        ell, elt = a.shape[1], _elt(self.N, step)
        ext = self.prepare(a, scale_c0=False)

        def call(pre, key, ind):
            out = np.empty((2, ell, self.N), dtype=np.uint64)
            work = np.zeros(self.lib.emu_rotate_modup_work_bytes(self.be.h, ell) // 8, dtype=np.uint64)
            self.be._chk(getattr(self.lib, pre + "rotate_modup_prepared")(self.be.h, ell, _p(out), _p(a), _p(ext), C.c_uint64(elt),
                                                                           C.c_void_p(key(elt)), C.c_void_p(ind(elt)), _p(work)))
            return out
        return self.both(t, call)

    def modup_many(self, t, a, steps):
        ell, n = a.shape[1], len(steps)
        ext = self.prepare(a, scale_c0=True)
        elts = [_elt(self.N, s) for s in steps]

        def call(pre, key, ind):
            out = np.empty((n, 2, ell, self.N), dtype=np.uint64)
            work = np.zeros(self.lib.emu_rotate_modup_many_work_bytes(self.be.h, ell, n) // 8, dtype=np.uint64)
            self.be._chk(getattr(self.lib, pre + "rotate_modup_many")(self.be.h, ell, n, _p(out), _p(a), _p(ext), (C.c_uint64 * n)(*elts),
                                                                       _ptrs([key(e) for e in elts]), _ptrs([ind(e) for e in elts]), _p(work)))
            return out
        return self.both(t, call)

    def wsum(self, t, a, steps, nout, seed):
        orc, ell, n = self.orcs[t], a.shape[1], len(steps)
        ext = self.prepare(a, scale_c0=True)
        elts = [_elt(self.N, s) for s in steps]
        rng = np.random.default_rng(seed)
        enc = lambda v: orc.encode(np.array([v]), 2.0 ** 30, ell)
        wts = [[None if rng.random() < 0.2 else enc(WSUM_VALUES[rng.integers(len(WSUM_VALUES))]) for _ in range(n)] for _ in range(nout)]
        taps = [a, pc.rand_ct(orc, 2, ell, 900 + seed)]
        twts = [[enc(-1.0 - oi), None if oi % 2 else enc(0.25 * oi + 0.5)] for oi in range(nout)]
        ptr = lambda w: None if w is None else w.ctypes.data

        def call(pre, key, ind):
            out = np.empty((nout, 2, ell, self.N), dtype=np.uint64)
            work = np.zeros(self.lib.emu_rotate_wsum_work_bytes(self.be.h, ell, n, nout) // 8, dtype=np.uint64)
            self.be._chk(getattr(self.lib, pre + "rotate_wsum")(self.be.h, ell, nout, _p(out), _p(a), _p(ext), n, (C.c_uint64 * n)(*elts),
                                                                 _ptrs([key(e) for e in elts]), _ptrs([ind(e) for e in elts]),
                                                                 _ptrs([ptr(w) for ws in wts for w in ws]), len(taps),
                                                                 _ptrs([x.ctypes.data for x in taps]), _ptrs([ptr(w) for ws in twts for w in ws]),
                                                                 _p(work)))
            return out
        got, want = self.both(t, call)
        return got, want, (wts, taps, twts)


CHAINS = {
    "60bit_4096": (4096, [60, 60, 60, 60, 60]),
    "mixed60_40_50": (1024, [60, 40, 50, 60]),
    "k6": (1024, [60, 50, 60, 50, 50, 60]),
}
STEPS = WSUM_STEPS        # 16 distinct elements


@pytest.fixture(scope="module", params=sorted(CHAINS))
def case(request):
    N, bits = CHAINS[request.param]
    return Case(N, bits, STEPS if N == 1024 else STEPS[:4])


def test_drawn_words_are_np_expand(case):
    """every (J, row) c1 row the seeded bodies draw, the P row included, is np_expand's"""
    b = case.banks
    for t in (0, 1):
        for e in [None] + case.elts[:2]:
            out = np.zeros((case.k - 1, case.k, case.N), dtype=np.uint64)
            img = b.seeded[t, b.sw * b.index(e):b.sw * (b.index(e) + 1)]
            case.be._chk(case.lib.emus_draw_c1(case.be.h, _p(img), _p(out)))
            assert np.array_equal(out, case.key(t, e)[:, 1])


@pytest.mark.parametrize("N", [1024, 2048])
def test_shared_draw_high_rejection_moduli(N):
    """the draw of the seeded bodies (kx_draw8) with the rule's % reducer: the acceptance test and the fallback search at rejection
    rates of 15 % to 40 %"""
    be = SeededEmu(1024, o.Oracle(1024, [60, 60]).primes)
    k = len(HIGH_REJECTION)
    q = np.array(HIGH_REJECTION, dtype=np.uint64)
    for sd in seeds_for(2, 99 + N):
        got = np.zeros((k - 1, k, N), dtype=np.uint64)
        buf = np.frombuffer(sd, dtype=np.uint8).copy()
        be._chk(be.lib.emus_draw_rows_rem(C.c_void_p(buf.ctypes.data), k, C.c_uint32(N), _p(q), _p(got)))
        want, fell = np_expand(sd, N, HIGH_REJECTION)
        assert fell.sum() > 0
        assert np.array_equal(got, want)


def test_barrett_reduction_equals_rem_on_ring_primes():
    """the seeded draw reduces an accepted candidate with barrett64: the value of % for every 64-bit input (edges and random)"""
    primes = o.Oracle(1024, [60, 40, 50, 30, 60]).primes
    be = SeededEmu(1024, primes)
    rng = np.random.default_rng(5)
    for m, p in enumerate(primes):
        p = int(p)
        lim = p * ((2 ** 64 - 1) // p)
        v = np.concatenate([rng.integers(0, 2 ** 63, 4000, dtype=np.uint64) * np.uint64(2) + np.uint64(1),
                            np.array([0, 1, p - 1, p, p + 1, 2 * p - 1, lim - 1, lim - p, 2 ** 64 - 1], dtype=np.uint64)])
        out = np.zeros_like(v)
        be._chk(be.lib.emus_barrett_vs_rem(be.h, m, _p(v), len(v), _p(out)))
        assert np.array_equal(out, v % np.uint64(p)), m


@pytest.mark.parametrize("t", [0, 1])
def test_relinearize_and_rotate_seeded_equal_expanded(case, t):
    orc = case.orcs[t]
    for ell in range(1, case.k):
        a3 = pc.rand_ct(orc, 3, ell, 40 * ell + t)
        got, want = case.relinearize(t, a3)
        pc.eq(got, want)
        a = pc.rand_ct(orc, 2, ell, 60 * ell + t)
        got, want = case.rotate(t, a, STEPS[1])
        pc.eq(got, want)
    ell = case.k - 1
    pc.eq(got, orc.rotate(a, STEPS[1], case.key(t, _elt(case.N, STEPS[1]))))


@pytest.mark.parametrize("t", [0, 1])
def test_rotate_modup_prepared_seeded_equals_expanded(case, t):
    orc = case.orcs[t]
    for ell in range(1, case.k):
        a = pc.rand_ct(orc, 2, ell, 100 * ell + t)
        for s in STEPS[:2]:
            got, want = case.modup_prepared(t, a, s)
            pc.eq(got, want)
    pc.eq(got, orc.rotate(a, STEPS[1], case.key(t, _elt(case.N, STEPS[1]))))


@pytest.mark.parametrize("t", [0, 1])
@pytest.mark.parametrize("n", [1, 3, 16])
def test_rotate_modup_many_seeded_equals_expanded(case, t, n):
    if n > len(case.steps):
        pytest.skip("the N = 4096 chain keys 4 elements")
    orc = case.orcs[t]
    for ell in range(1, case.k):
        a = pc.rand_ct(orc, 2, ell, 300 + 10 * ell + n + t)
        got, want = case.modup_many(t, a, STEPS[:n])
        pc.eq(got, want)
    for i, s in enumerate(STEPS[:min(n, 3)]):
        pc.eq(got[i], orc.rotate(a, s, case.key(t, _elt(case.N, s))))


@pytest.mark.parametrize("t", [0, 1])
@pytest.mark.parametrize("nout", [1, 2, 3, 4])
def test_rotate_wsum_seeded_equals_expanded(case, t, nout):
    orc = case.orcs[t]
    for ell in range(1, case.k):
        n = min((5, 16, 8, 3)[ell % 4], len(case.steps))
        a = pc.rand_ct(orc, 2, ell, 500 + 10 * ell + nout + t)
        got, want, (wts, taps, twts) = case.wsum(t, a, STEPS[:n], nout, seed=ell * 7 + nout)
        pc.eq(got, want)
    rots = [orc.rotate(a, s, case.key(t, _elt(case.N, s))) for s in STEPS[:n]]
    for oi in range(nout):
        acc = None
        for c_, w in list(zip(rots, wts[oi])) + list(zip(taps, twts[oi])):
            if w is not None:
                term = orc.mul_plain(c_, w)
                acc = term if acc is None else orc.add(acc, term)
        pc.eq(got[oi], acc)


def test_tenants_differ():
    """the key-bank offset moves the seed with the c0 rows: tenant 1's words are its own"""
    c = Case(*CHAINS["mixed60_40_50"], STEPS[:4], salt=3)
    a = pc.rand_ct(c.orcs[0], 2, 2, 9)
    outs = []
    for t in (0, 1):
        got, want = c.modup_many(t, a, STEPS[:4])
        pc.eq(got, want)
        outs.append(got)
    assert not np.array_equal(outs[0], outs[1])


@pytest.fixture(scope="module")
def small():
    return Case(*CHAINS["mixed60_40_50"], STEPS[:2], salt=7)


def test_lazy_rotsum_refuses_seeded(small):
    c, ell = small, 2
    a = pc.rand_ct(c.orcs[0], 2, ell, 3)
    ext = c.prepare(a, scale_c0=True)
    elts = [_elt(c.N, s) for s in STEPS[:2]]
    work = np.zeros(c.lib.emu_lazy_rotsum_work_bytes(c.be.h, ell, 1) // 8, dtype=np.uint64)
    wt = np.zeros((ell + 1, c.N), dtype=np.uint64)
    out = np.empty((1, 2, ell, c.N), dtype=np.uint64)
    rc = c.lib.emus_lazy_rotsum(c.be.h, ell, 1, _p(out), _p(a), _p(ext), 2, (C.c_uint64 * 2)(*elts), _ptrs([c.banks.seeded_key(e) for e in elts]),
                                _ptrs([c.banks.ind_ptr(e) for e in elts]), _ptrs([wt.ctypes.data, wt.ctypes.data]), _p(work))
    assert rc != 0 and b"lazy_rotsum" in c.lib.emu_last_error()


def test_hoist_constants_refuse_seeded(small):
    c = small
    out = np.zeros(1, dtype=np.uint64)
    rc = c.lib.emus_rotate_hoist_const(c.be.h, 1, C.c_uint64(c.elts[0]), _p(c.banks.seeded), _p(out), _p(out))
    assert rc != 0 and b"evab_set_key_seeded" in c.lib.emu_last_error()


def test_hoisted_calls_refuse_seeded_without_inline(small):
    c = small
    a = pc.rand_ct(c.orcs[0], 2, 2, 4)
    try:
        c.lib.emus_set_hoist_inline(0)
        with pytest.raises(Exception, match="inline hoist constants"):
            c.modup_prepared(0, a, STEPS[0])
        with pytest.raises(Exception, match="inline hoist constants"):
            c.modup_many(0, a, STEPS[:2])
    finally:
        c.lib.emus_set_hoist_inline(1)
