"""Cached c1 rows of a seeded key bank (evab_set_key_c1_rows, evab_expand_seeded_c1, B200Server(c1_cache=H)) on the CPU: the key
switches of an instance with a c1 region read its rows from the region (tests/emu/emu_c1cache.cpp replays the SEED bodies with the
tile copied from the region) and equal, word for word, the same ops on the expanded keys -- and the drawing instances still do --
at every level, for two tenants, on the chains of test_seeded_slots.py; the expansion body writes np_expand's rows in the region
geometry; the calls refuse a region table without seeded keys or a key-bank table; and the admission and eviction policy (host
C1Cache) against a small Python model."""
import ctypes as C

import numpy as np
import pytest

import parity_cases as pc
from backends import _elt, _p
from oracle import oracle as o
from test_seeded_slots import CHAINS, STEPS, Banks, Case, SeededEmu


class C1Emu(SeededEmu):
    """the seeded emulator with the cached-row replays (emuc_*)"""
    SRC, LIB = "emu_c1cache.cpp", "libevab_emu_c1cache"


class C1Case(Case):
    """two tenants in bank slots 0 and 1 of a seeded bank with two c1 regions (bank regions 2 and 3) after them, region 2 + t holding
    tenant t's expanded c1 rows.  `region` is the c1 table entry of the replayed instance: -1 draws"""

    def __init__(self, N, bits, steps, salt=0):
        self.orcs = [o.Oracle(N, bits).keygen(seed) for seed in (31, 32)]
        self.be = C1Emu(N, self.orcs[0].primes)
        self.N, self.k, self.lib = N, self.be.k, self.be.lib
        self.steps = list(steps)
        self.elts = sorted({_elt(N, s) for s in self.steps})
        self.banks = Banks(self.be, self.orcs, self.elts, salt + N + len(bits))
        self.table = np.zeros(1, dtype=np.int32)
        self.c1tab = np.full(1, -1, dtype=np.int32)
        b = self.banks
        self.stride = b.seeded.shape[1]
        self.nk = 1 + len(self.elts)
        self.bank = np.zeros((4, self.stride), dtype=np.uint64)
        self.bank[:2] = b.seeded
        for t in (0, 1):
            self.be._chk(self.lib.emuc_expand_seeded_c1(self.be.h, self.nk, _p(self.bank[t]), _p(self.bank[2 + t])))
        self.region = -1

    def c1_key(self, e):
        return self.bank.ctypes.data + 8 * self.banks.sw * self.banks.index(e)

    def both(self, t, call, exp_prefix="emui_"):
        b = self.banks
        try:
            self.select(t, b.exp.shape[1])
            want = call(exp_prefix, b.exp_key, b.ind_ptr)
            self.select(t, self.stride)
            self.c1tab[0] = self.region
            self.lib.emuc_set_key_c1_rows(self.c1tab.ctypes.data_as(C.c_void_p))
            got = call("emuc_", self.c1_key, b.ind_ptr)
        finally:
            self.lib.emuc_set_key_c1_rows(None)
            self.lib.emu_set_key_bank(None, C.c_size_t(0))
        return got, want


@pytest.fixture(scope="module", params=sorted(CHAINS))
def case(request):
    N, bits = CHAINS[request.param]
    return C1Case(N, bits, STEPS if N == 1024 else STEPS[:4])


def regions_of(t):
    """the two ways tenant t's instance can run: from its region, and drawing"""
    return [2 + t, -1]


def test_expand_writes_np_expand_rows_in_region_geometry(case):
    """key i's c1 rows [k-1][k][N] sit where its c0 rows sit in a seeded image; the 8 seed words stay untouched"""
    b, sw = case.banks, case.banks.sw
    for t in (0, 1):
        reg = case.bank[2 + t]
        for e in [None] + case.elts:
            i = b.index(e)
            rows = reg[sw * i:sw * i + sw - 8].reshape(case.k - 1, case.k, case.N)
            assert np.array_equal(rows, case.key(t, e)[:, 1])
            assert not reg[sw * i + sw - 8:sw * (i + 1)].any()


@pytest.mark.parametrize("t", [0, 1])
def test_relinearize_and_rotate_cached_equal_expanded(case, t):
    orc = case.orcs[t]
    for region in regions_of(t):
        case.region = region
        for ell in range(1, case.k):
            a3 = pc.rand_ct(orc, 3, ell, 40 * ell + t)
            got, want = case.relinearize(t, a3)
            pc.eq(got, want)
            a = pc.rand_ct(orc, 2, ell, 60 * ell + t)
            got, want = case.rotate(t, a, STEPS[1])
            pc.eq(got, want)
        pc.eq(got, orc.rotate(a, STEPS[1], case.key(t, _elt(case.N, STEPS[1]))))


@pytest.mark.parametrize("t", [0, 1])
def test_rotate_modup_prepared_cached_equals_expanded(case, t):
    orc = case.orcs[t]
    for region in regions_of(t):
        case.region = region
        for ell in range(1, case.k):
            a = pc.rand_ct(orc, 2, ell, 100 * ell + t)
            for s in STEPS[:2]:
                got, want = case.modup_prepared(t, a, s)
                pc.eq(got, want)
        pc.eq(got, orc.rotate(a, STEPS[1], case.key(t, _elt(case.N, STEPS[1]))))


@pytest.mark.parametrize("t", [0, 1])
@pytest.mark.parametrize("n", [1, 3, 16])
def test_rotate_modup_many_cached_equals_expanded(case, t, n):
    if n > len(case.steps):
        pytest.skip("the N = 4096 chain keys 4 elements")
    orc = case.orcs[t]
    for region in regions_of(t):
        case.region = region
        for ell in range(1, case.k):
            a = pc.rand_ct(orc, 2, ell, 300 + 10 * ell + n + t)
            got, want = case.modup_many(t, a, STEPS[:n])
            pc.eq(got, want)
        for i, s in enumerate(STEPS[:min(n, 3)]):
            pc.eq(got[i], orc.rotate(a, s, case.key(t, _elt(case.N, s))))


@pytest.mark.parametrize("t", [0, 1])
@pytest.mark.parametrize("nout", [1, 2, 3, 4])
def test_rotate_wsum_cached_equals_expanded(case, t, nout):
    orc = case.orcs[t]
    for region in regions_of(t):
        case.region = region
        for ell in range(1, case.k):
            n = min((5, 16, 8, 3)[ell % 4], len(case.steps))
            a = pc.rand_ct(orc, 2, ell, 500 + 10 * ell + nout + t)
            got, want, _ = case.wsum(t, a, STEPS[:n], nout, seed=ell * 7 + nout)
            pc.eq(got, want)


def test_region_rows_are_read():
    """an instance pointed at the other tenant's region switches with that tenant's c1 rows: the table is what selects them"""
    c = C1Case(*CHAINS["mixed60_40_50"], STEPS[:4], salt=3)
    a = pc.rand_ct(c.orcs[0], 2, 2, 9)
    c.region = 2
    good, want = c.modup_many(0, a, STEPS[:4])
    pc.eq(good, want)
    c.region = 3
    bad, _ = c.modup_many(0, a, STEPS[:4])
    assert not np.array_equal(bad, want)
    c.region = -1


@pytest.fixture(scope="module")
def small():
    return C1Case(*CHAINS["mixed60_40_50"], STEPS[:2], salt=7)


def test_c1_rows_refuse_without_seeded_keys(small):
    c = small
    a = pc.rand_ct(c.orcs[0], 2, 2, 4)
    c.region = 2
    try:
        c.lib.emuc_set_key_seeded(0)
        with pytest.raises(Exception, match="evab_set_key_seeded"):
            c.rotate(0, a, STEPS[0])
        with pytest.raises(Exception, match="evab_set_key_seeded"):
            c.modup_many(0, a, STEPS[:2])
    finally:
        c.lib.emuc_set_key_seeded(1)
        c.region = -1


def test_c1_rows_refuse_without_key_bank(small):
    c = small
    a = pc.rand_ct(c.orcs[0], 2, 2, 5)
    out = np.empty((2, 2, c.N), dtype=np.uint64)
    work = np.zeros(c.lib.emu_keyswitch_work_bytes(c.be.h, 2) // 8 + 8 * c.N * 4, dtype=np.uint64)
    tab = np.zeros(1, dtype=np.int32)
    try:
        c.lib.emuc_set_key_c1_rows(tab.ctypes.data_as(C.c_void_p))
        rc = c.lib.emuc_relinearize(c.be.h, 2, _p(out), _p(pc.rand_ct(c.orcs[0], 3, 2, 6)), C.c_void_p(c.c1_key(None)), _p(work))
        assert rc != 0 and b"evab_set_key_bank" in c.lib.emu_last_error()
        rc = c.lib.emuc_rotate(c.be.h, 2, _p(out), _p(a), C.c_uint64(c.elts[0]), C.c_void_p(c.c1_key(c.elts[0])), _p(work))
        assert rc != 0 and b"evab_set_key_bank" in c.lib.emu_last_error()
    finally:
        c.lib.emuc_set_key_c1_rows(None)


# ---- admission and eviction (host/slot_cache.hpp C1Cache) ---------------------------------------------------------------------

class C1Model:
    """admission: more instances first, ties by first appearance, the first `regions` admitted; admitted tenants holding a region are
    pinned; a missing admitted one takes the lowest free region, else the least recently used unpinned one; every instance whose
    tenant then holds a region reads it"""

    def __init__(self, regions):
        self.R = regions
        self.owner, self.stamp, self.region = [-1] * regions, [0] * regions, {}
        self.clock = self.fills = self.evictions = 0

    def assign(self, tenants):
        first = list(dict.fromkeys(tenants))
        admitted = sorted(first, key=lambda t: -tenants.count(t))[:self.R]   # sorted() is stable: ties keep first appearance
        pinned = {self.region[t] for t in admitted if t in self.region}
        fills = []
        for t in admitted:
            if t in self.region:
                continue
            free = [r for r in range(self.R) if self.owner[r] < 0]
            r = free[0] if free else min((r for r in range(self.R) if r not in pinned), key=lambda r: self.stamp[r])
            old = self.owner[r]
            if old >= 0:
                del self.region[old]
                self.evictions += 1
            self.owner[r], self.region[t] = t, r
            pinned.add(r)
            fills.append((t, r, old))
            self.fills += 1
        self.clock += 1
        for t in tenants:
            if t in self.region:
                self.stamp[self.region[t]] = self.clock
        return [self.region.get(t, -1) for t in tenants], fills, [t for t in self.owner if t >= 0]

    def drop(self, t):
        if t in self.region:
            r = self.region.pop(t)
            self.owner[r], self.stamp[r] = -1, 0


def replay_model(regions, ops):
    m = C1Model(regions)
    out = []
    for op in ops:
        if isinstance(op, tuple):
            m.drop(op[1])
            out.append(None)
        else:
            out.append(m.assign(op))
    return out, m.fills, m.evictions


def replay_native(regions, ops):
    from eva_b200 import _eva_b200 as native
    res, fills, ev = native._c1_cache(regions, ops)
    norm = [None if r is None else (list(r[0]), [tuple(f) for f in r[1]], list(r[2])) for r in res]
    return norm, fills, ev


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("regions", [1, 2, 3, 5])
def test_c1_cache_matches_model(seed, regions):
    rng = np.random.default_rng(500 * regions + seed)
    ops = []
    for _ in range(60):
        if rng.random() < 0.08:
            ops.append(("remove", int(rng.integers(0, 12))))
        else:
            n = int(rng.integers(1, 3 * regions + 3))
            hot = int(rng.integers(1, 13))
            ops.append([int(t) for t in rng.integers(0, hot, n)])
    assert replay_native(regions, ops) == replay_model(regions, ops)


def test_c1_cache_admits_by_count_then_first_appearance():
    res, fills, ev = replay_native(2, [[5, 7, 7, 9, 9, 9], [1, 2, 1, 2, 3, 3, 3]])
    # 9 (3 instances), then 7 (2): 5 draws
    assert res[0] == ([-1, 1, 1, 0, 0, 0], [(9, 0, -1), (7, 1, -1)], [9, 7])
    # 3 leads; 1 and 2 tie at 2 and 1 appears first: 9 and 7 (least recently used alike) are evicted in region order
    assert res[1] == ([1, -1, 1, -1, 0, 0, 0], [(3, 0, 9), (1, 1, 7)], [3, 1])
    assert (fills, ev) == (4, 2)


def test_c1_cache_pins_admitted_and_keeps_unadmitted_hits():
    res, _, _ = replay_native(2, [[0, 1], [2, 2, 0, 1], [1, 2, 2, 3, 3, 3]])
    # 2 and 0 admitted: 0 is pinned, 2 takes 1's region; 1 was not admitted and lost its region
    assert res[1] == ([1, 1, 0, -1], [(2, 1, 1)], [0, 2])
    # 3 then 2 admitted (2 pinned); 3 evicts 0; 1 holds nothing and draws
    assert res[2] == ([-1, 1, 1, 0, 0, 0], [(3, 0, 0)], [3, 2])
    res, _, _ = replay_native(2, [[0, 1], [0, 0, 2, 2, 1]])
    # 0 and 2 admitted; 2 evicts 1 (the least recently used unpinned region)
    assert res[1] == ([0, 0, 1, 1, -1], [(2, 1, 1)], [0, 2])
    res, _, _ = replay_native(3, [[0, 1, 2], [3, 3, 4, 4, 0]])
    # all three admitted, 0 pinned: 3 and 4 take the regions of 1 and 2 (same stamp: the lowest region first)
    assert res[1] == ([1, 1, 2, 2, 0], [(3, 1, 1), (4, 2, 2)], [0, 3, 4])


def test_c1_cache_more_tenants_than_regions_and_repeat():
    res, fills, ev = replay_native(1, [[4, 5, 6, 7], [4, 5, 6, 7], [4, 5, 6, 7]])
    assert res[0] == ([0, -1, -1, -1], [(4, 0, -1)], [4])
    assert res[1] == res[2] == ([0, -1, -1, -1], [], [4])   # a repeated batch fills nothing
    assert (fills, ev) == (1, 0)


def test_c1_cache_drop_frees_the_region():
    res, fills, ev = replay_native(2, [[0, 1], ("remove", 0), [0], [2]])
    assert res[1] is None
    assert res[2] == ([0], [(0, 0, -1)], [0, 1])   # the id is filled again, from the new keys' seeds
    assert res[3] == ([1], [(2, 1, 1)], [0, 2])
    assert (fills, ev) == (4, 1)
