"""Paged evaluation keys: B200Server(max_tenants > capacity) keeps every tenant's keys in page-locked host memory and pages them
into the key bank's device slots as batches need them; every output is checked against the oracle run with that instance's own
keys.  Also the one-pass hoist constants of every level (evab_rotate_hoist_const_levels) against the one-level call."""
import copy
import ctypes as C

import numpy as np
import pytest

from backends import GpuBackend, _p
from oracle import oracle as o
from test_slot_cache import LruModel

# ---------------------------------------------------------------------------------------------------------------------------
# evab_rotate_hoist_const_levels == evab_rotate_hoist_const for every (element, level)


def _levels_vs_one_level(orc, steps):
    N, k = orc.N, orc.k
    be = GpuBackend(N, orc.primes)
    lib = be.lib
    elts = [o.galois_elt_from_step(N, s) for s in steps]
    for e in elts:
        be._chk(lib.evab_galois_prepare(be.h, C.c_uint64(e)))
    keys = np.stack([orc.galois_key(e) for e in elts])
    dk = be._up(keys)
    per = lib.evab_hoist_const_levels_bytes(be.h)
    assert per == 8 * ((k + 1) * k - 2) * N
    out = be._alloc(len(elts) * per)
    tmp = be._alloc(lib.evab_rotate_hoist_const_levels_work_bytes(be.h, len(elts)))
    ea = (C.c_uint64 * len(elts))(*elts)
    be._chk(lib.evab_rotate_hoist_const_levels(be.h, len(elts), ea, dk, out, tmp, None))
    got = be._down(out, (len(elts), per // 8))
    one = be._alloc(lib.evab_hoist_const_bytes(be.h, k - 1))
    otmp = be._alloc(8 * k * N)
    for g, e in enumerate(elts):
        off = 0
        for ell in range(1, k):
            w = 2 * (ell + 1) * N
            key_g = C.c_void_p(dk.value + g * keys[0].nbytes)
            be._chk(lib.evab_rotate_hoist_const(be.h, ell, C.c_uint64(e), key_g, one, otmp, None))
            want = be._down(one, (w,))
            assert np.array_equal(got[g, off:off + w], want), (N, k, e, ell)
            off += w
    for d in (dk, out, tmp, one, otmp):
        lib.evab_free(be.h, d, None)


@pytest.mark.gpu
def test_levels_equal_one_call_per_level_sobel_shape():
    """N = 16384, five 60-bit primes, Sobel's nine rotation steps"""
    orc = o.Oracle(16384, [60] * 5).keygen(1)
    _levels_vs_one_level(orc, (1, 2, 64, 65, 66, 128, 129, 130, -1))


@pytest.mark.gpu
def test_levels_equal_one_call_per_level_seal14():
    """the 14-prime SEAL-scan chain at N = 32768: 13 levels, sums of up to 13 terms"""
    orc = o.Oracle(32768, primes=o.gen_primes(32768, [60] * 14)).keygen(3)
    _levels_vs_one_level(orc, (1, -5))


# ---------------------------------------------------------------------------------------------------------------------------
# B200Server with paging, against the oracle with each instance's own keys

SEEDS = tuple(range(1, 8))      # 7 tenants, max_tenants = 8
INSTANCES = 4


class PagedFixture:
    """a golden program; 7 tenants with oracle keys of seeds 1..7; servers with max_tenants = 8 and `capacity` device slots"""

    def __init__(self, name):
        from eva_b200 import b200, program_io as gl
        from oracle_exec import OracleProgram
        self.d = d = gl.load_json(name)
        self.prog, self.params, _, self.terms = gl.build_program(d)
        self.N = d["poly_modulus_degree"]
        probe = b200.B200Server(self.params, capacity=1)
        self.elts = probe.bank_info()["galois_elements"]
        del probe
        self.orcs, self.ops, self.keys = [], [], []
        for seed in SEEDS:
            orc = o.Oracle(self.N, d["prime_bits"]).keygen(seed)
            op = OracleProgram(d, orc)
            op.prepare_keys()
            op.gks.update({e: orc.galois_key(e) for e in self.elts if e not in op.gks})
            self.orcs.append(orc); self.ops.append(op)
            self.keys.append((op.rk, {int(e): op.gks[e] for e in self.elts}))
        self.vals, self.ins = [], []
        for i in range(INSTANCES):
            v, io = self.valuation(self.orcs[i % len(self.orcs)], seed=40 + i)
            self.vals.append(v); self.ins.append(io)
        self._want = {}

    def server(self, capacity, max_tenants=8):
        from eva_b200 import b200
        s = b200.B200Server(self.params, capacity=capacity, max_tenants=max_tenants)
        for t in range(len(SEEDS)):
            assert s.add_raw_keys(*self.keys[t]) == t
        info = s.bank_info()
        assert info["device_slots"] == capacity and info["max_tenants"] == max_tenants and info["resident"] == []
        assert info["fills"] == 0 and info["host_key_bytes"] == len(SEEDS) * info["key_bytes_per_tenant"]
        return s

    def valuation(self, orc, seed):
        from eva_b200 import b200
        rng = np.random.default_rng(seed)
        val, io = b200.B200Valuation(), {}
        for name_, info in self.d["signature"].items():
            x = rng.uniform(0.0, 0.2, self.d["vec_size"])
            ell, scale = orc.k - 1 - info["level"], 2.0 ** info["scale"]
            if info["type"] == "Cipher":
                ct = orc.encrypt(orc.encode(x, scale, ell), seed=seed)
                val.set_cipher(name_, ct, scale); io[name_] = ("cipher", ct, scale)
            elif info["type"] == "Raw":
                val.set_raw(name_, list(x)); io[name_] = ("raw", x)
            else:
                pt = orc.encode(x, scale, ell)
                val.set_plain(name_, pt, scale); io[name_] = ("plain", pt, scale)
        return val, io

    def want(self, i, t):
        if (i, t) not in self._want:
            self._want[(i, t)] = self.ops[t].run(self.ins[i])
        return self._want[(i, t)]

    def check(self, outs, assign, what):
        assert len(outs) == len(assign)
        for i, (out, t) in enumerate(zip(outs, assign)):
            V = self.want(i, t)
            for oname, oid in self.d["outputs"].items():
                kind, arr, scale = out.get(oname)
                if kind == "cipher":
                    assert np.array_equal(arr, V[oid][1]) and scale == V[oid][2], (what, i, t, oname)

    def requests(self, assign):
        return list(zip(assign, self.vals))


def _assignments(rng, capacity, count):
    """batches of INSTANCES instances naming at most `capacity` distinct tenants, drawn so that hits, misses and evictions mix"""
    out = []
    for _ in range(count):
        pool = [int(t) for t in rng.choice(len(SEEDS), size=int(rng.integers(1, capacity + 1)), replace=False)]
        out.append([pool[int(j)] for j in rng.integers(0, len(pool), INSTANCES)])
    return out


_FIX = {}


def fixture(name):
    if name not in _FIX:
        _FIX[name] = PagedFixture(name)
    return _FIX[name]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["sobel", "harris", "polynomial", "feat_mixed"])
def test_paged_batches_bit_exact(name):
    """capacity 2 and 3 with 7 tenants: 5 seeded execute_batch calls each, mixed assignments; every output is the oracle's with the
    instance's own keys, fills and evictions are the policy model's, and no plan is built after the first batch"""
    f = fixture(name)
    for capacity in (2, 3):
        s = f.server(capacity)
        model = LruModel(capacity)
        rng = np.random.default_rng(100 * capacity + len(name))
        built = None
        for n, assign in enumerate(_assignments(rng, capacity, 5)):
            f.check(s.execute_batch(f.prog, f.requests(assign)), assign, (name, capacity, n))
            model.assign(assign)
            info = s.bank_info()
            assert (info["fills"], info["evictions"]) == (model.fills, model.evictions), (name, capacity, n)
            assert sorted(info["resident"]) == sorted(t for t in model.owner if t >= 0)
            if built is None:
                built = s.plans_built()
            assert s.plans_built() == built
        assert model.evictions > 0


@pytest.mark.gpu
def test_paged_async_batches_evicting_each_other():
    """two execute_batch_async batches in different submit slots, the second evicting every slot the first reads: both exact"""
    f = fixture("sobel")
    s = f.server(2)
    a, b = [0, 1, 0, 1], [2, 3, 3, 2]
    for _ in range(2):
        ha = s.execute_batch_async(f.prog, f.requests(a), 0)
        hb = s.execute_batch_async(f.prog, f.requests(b), 1)
        f.check(s.execute_batch_result(ha), a, "first")
        f.check(s.execute_batch_result(hb), b, "second")
    assert s.bank_info()["evictions"] >= 6


@pytest.mark.gpu
def test_paged_zero_digit_redo_refills_an_evicted_tenant():
    """an instance of tenant 1 holds a zero digit coefficient: its batch is redone at collect, after another batch evicted tenant
    1 and 2; the redo fills them again and both batches are exact"""
    from eva_b200 import b200
    f = copy.copy(fixture("sobel"))     # its own inputs and expected values; the keys and oracles are shared
    f.vals, f.ins, f._want = list(f.vals), list(f.ins), {}
    s = f.server(2)
    (name_, info), = f.d["signature"].items()
    orc = f.orcs[1]
    ell = orc.k - 1 - info["level"]
    ct = f.ins[1][name_][1].copy()
    c1 = np.stack([orc.ntt_inv(ct[1, r], r) for r in range(ell)])
    c1[1, 7] = 0
    ct[1] = np.stack([orc.ntt_fwd(c1[r], r) for r in range(ell)])
    f.vals[1] = b200.B200Valuation()
    f.vals[1].set_cipher(name_, ct, 2.0 ** info["scale"])
    f.ins[1] = {name_: ("cipher", ct, 2.0 ** info["scale"])}
    a, b = [2, 1, 2, 1], [3, 4, 4, 3]
    ha = s.execute_batch_async(f.prog, f.requests(a), 0)
    hb = s.execute_batch_async(f.prog, f.requests(b), 1)
    assert sorted(s.bank_info()["resident"]) == [3, 4]
    fills = s.bank_info()["fills"]
    f.check(s.execute_batch_result(ha), a, "redo")
    assert s.bank_info()["fills"] == fills + 2 and sorted(s.bank_info()["resident"]) == [1, 2]
    f.check(s.execute_batch_result(hb), b, "other")


@pytest.mark.gpu
def test_paged_errors():
    from eva_b200 import b200
    f = fixture("polynomial")
    with pytest.raises(Exception, match="below"):
        b200.B200Server(f.params, capacity=3, max_tenants=2)
    s = f.server(2)
    rk, gks = f.keys[0]
    # too many distinct tenants for the slots: both numbers in the message, nothing filled
    with pytest.raises(Exception, match="3 distinct tenants.*2 device slots"):
        s.execute_batch(f.prog, f.requests([0, 1, 2, 0]))
    assert s.bank_info()["fills"] == 0
    # the host store: 8 ids, 7 used
    assert s.add_raw_keys(rk, gks) == 7
    with pytest.raises(Exception, match="host key store is full"):
        s.add_raw_keys(rk, gks)
    # unknown tenants
    for bad in (8, -1):
        with pytest.raises(Exception):
            s.execute(f.prog, bad, f.vals[0])
    s.remove_keys(7)
    with pytest.raises(Exception, match="no keys"):
        s.execute(f.prog, 7, f.vals[0])
    # removing a tenant an uncollected batch uses; then removal frees its slot and its id
    h = s.execute_batch_async(f.prog, f.requests([0, 1, 0, 1]), 0)
    with pytest.raises(Exception, match="not been collected"):
        s.remove_keys(1)
    f.check(s.execute_batch_result(h), [0, 1, 0, 1], "async")
    s.remove_keys(1)
    assert 1 not in s.bank_info()["resident"] and s.bank_info()["tenants"] == 6
    assert s.add_raw_keys(*f.keys[1]) == 1
    f.check(s.execute_batch(f.prog, f.requests([1, 0, 1, 0])), [1, 0, 1, 0], "re-added")
    # max_tenants == capacity: today's server (tenant id = slot, full past capacity)
    same = b200.B200Server(f.params, capacity=2, max_tenants=2)
    same.add_raw_keys(rk, gks); same.add_raw_keys(rk, gks)
    with pytest.raises(Exception, match="key bank is full"):
        same.add_raw_keys(rk, gks)
    assert same.bank_info()["resident"] == [0, 1] and same.bank_info()["fills"] == 2
