"""Cached c1 rows on the GPU: evab_set_key_c1_rows / evab_expand_seeded_c1 at the C-ABI, and B200Server(key_storage="seeded",
c1_cache=H).  An instance with a c1 region reads its keys' c1 rows from it, the others draw them; either way the outputs equal, byte
for byte, a c1_cache=0 seeded server and an expanded inline server -- Sobel and Harris with 3 tenants, fuse 1 and 3, power-of-two
keys with paging, sync and async, a bank-slot eviction and refill, remove_keys and a reused id, the zero-digit redo -- and the
counters and the error cases are as documented."""
import ctypes as C

import numpy as np
import pytest

import parity_cases as pc
from backends import _elt
from oracle import oracle as o
from test_rotation_wsum import WSUM_VALUES, _ptrs
from test_seeded_slots_gpu import ASSIGN, SeededGpu, _inputs, _load, _same

pytestmark = pytest.mark.gpu


# ---- the C-ABI: every seeded call with a cached and a drawing c1 table entry against the expanded key

class C1Gpu(SeededGpu):
    """SeededGpu plus a four-region seeded bank per key: [decoy image, image, c1 rows of the decoy, c1 rows of the image], the c1
    rows written by evab_expand_seeded_c1.  The instance reads region 1 (tenant table) and, through the c1 table, region 3 (cached)
    or nothing (-1, drawn)"""

    def __init__(self, orc, names, salt):
        super().__init__(orc, names, salt)
        sw = self.sw
        self.c1bank, self.rows = {}, {}
        for name in names:
            pair = self._down(self.dev[name][("seeded", True)], (2 * sw,))
            d = self._up(np.concatenate([pair, np.zeros(2 * sw, dtype=np.uint64)]))
            self._chk(self.lib.evab_expand_seeded_c1(self.h, 2, d, C.c_void_p(d.value + 16 * sw), None))
            self.c1bank[name] = d
            self.rows[name] = self._down(d, (4, sw))[3]
        self.c1tab = {r: self._up(np.array([r & 0xFFFFFFFF], dtype=np.uint64)) for r in (3, -1)}

    def modes(self, fn):
        out = super().modes(fn)
        lib = self.lib
        for r, tab in self.c1tab.items():
            self._chk(lib.evab_set_key_bank(self.table, C.c_size_t(self.sw)))
            self._chk(lib.evab_set_hoist_inline(1))
            self._chk(lib.evab_set_key_seeded(1))
            self._chk(lib.evab_set_key_c1_rows(tab))
            try:
                out[("c1", r)] = fn(lambda name: self.c1bank[name])
            finally:
                lib.evab_set_key_c1_rows(None)
                lib.evab_set_key_seeded(0)
                lib.evab_set_hoist_inline(0)
                lib.evab_set_key_bank(None, C.c_size_t(0))
        return out


def _all_equal(r):
    want = r[("expanded", False)]
    assert ("c1", 3) in r and ("c1", -1) in r
    for got in r.values():
        if isinstance(want, tuple):
            for g, w in zip(got, want):
                pc.eq(g, w)
        else:
            pc.eq(got, want)
    return want


def _cabi_c1_case(N, bits, steps, levels=None, salt=0):
    orc = o.Oracle(N, list(bits)).keygen(3)
    elts = [_elt(N, s) for s in steps]
    be = C1Gpu(orc, [None] + elts, salt + N + len(bits))
    for name in [None] + elts:   # evab_expand_seeded_c1 writes the expanded key's c1 rows where the image's c0 rows sit
        assert np.array_equal(be.rows[name][:be.sw - 8].reshape(orc.k - 1, orc.k, N), be.full[name][:, 1])
        assert not be.rows[name][be.sw - 8:].any()
    rng = np.random.default_rng(9)
    for ell in (levels or range(1, orc.k)):
        a3 = pc.rand_ct(orc, 3, ell, 20 + ell)
        relin = _all_equal(be.relinearize(a3))
        a = pc.rand_ct(orc, 2, ell, 40 + ell)
        plain, prepared = _all_equal(be.rotate(a, elts[0]))
        pc.eq(prepared, plain)
        pc.eq(_all_equal(be.modup_prepared(a, elts[0])), plain)
        pc.eq(_all_equal(be.modup_many(a, elts))[0], plain)
        enc = lambda v: orc.encode(np.array([v]), 2.0 ** 30, ell)
        y = pc.rand_ct(orc, 2, ell, 80 + ell)
        for nout in range(1, 5):
            wts = [[None if rng.random() < 0.2 else enc(WSUM_VALUES[rng.integers(len(WSUM_VALUES))]) for _ in elts] for _ in range(nout)]
            twts = [[enc(-1.0 - oi), None if oi % 2 else enc(0.5)] for oi in range(nout)]
            _all_equal(be.wsum(a, elts, wts, [a, y], twts))
        if ell == orc.k - 1:
            pc.eq(plain, orc.rotate(a, steps[0], be.full[elts[0]]))
            pc.eq(relin, orc.relinearize(a3, be.full[None]))
    return be


def test_cabi_c1_sobel_shape():
    _cabi_c1_case(16384, [60] * 5, [1, 64, 130])


def test_cabi_c1_mixed_chain():
    _cabi_c1_case(4096, [60, 50, 40, 50, 60], [1, -3, 7])


def test_cabi_c1_deep_chain():
    """14 primes: the 256-thread tiles of the cached instances pass the 48 KB shared-memory default at ell = 13"""
    _cabi_c1_case(4096, [60] + [50] * 12 + [60], [1, -3], levels=[1, 12, 13], salt=5)


def test_cabi_c1_refusals():
    orc = o.Oracle(4096, [60, 60, 60]).keygen(4)
    e = _elt(4096, 1)
    be = C1Gpu(orc, [None, e], 17)
    lib, ell = be.lib, 1
    a = pc.rand_ct(orc, 2, ell, 3)
    da, do = be._up(a), be._alloc(2 * ell * 4096 * 8)
    dw = be._alloc(lib.evab_keyswitch_work_bytes(be.h, ell))
    lib.evab_set_key_c1_rows(be.c1tab[3])
    try:
        lib.evab_set_key_bank(be.table, C.c_size_t(be.sw))
        rc = lib.evab_rotate(be.h, ell, do, da, C.c_uint64(e), be.c1bank[e], dw, None)
        assert rc != 0 and b"evab_set_key_seeded" in lib.evab_last_error()
        lib.evab_set_key_bank(None, C.c_size_t(0))
        lib.evab_set_key_seeded(1)
        rc = lib.evab_rotate(be.h, ell, do, da, C.c_uint64(e), be.dev[e][("seeded", False)], dw, None)
        assert rc != 0 and b"evab_set_key_bank" in lib.evab_last_error()
    finally:
        lib.evab_set_key_c1_rows(None)
        lib.evab_set_key_seeded(0)
        lib.evab_set_key_bank(None, C.c_size_t(0))
    be._free(da, do, dw)


# ---- B200Server(key_storage="seeded", c1_cache=H)

def _server(params, c1, **kw):
    from eva_b200 import b200
    if c1 is None:
        return b200.B200Server(params, hoist_constants="inline", key_storage="expanded", **kw)
    return b200.B200Server(params, hoist_constants="inline", key_storage="seeded", c1_cache=c1, **kw)


@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_server_c1_bit_exact(name):
    """3 tenants (two instances each), c1_cache 1, 2 and capacity: fuse 1 and 3, with and without rotation sums, without the shared
    mod-up: byte-equal to the c1_cache=0 seeded server and the expanded inline server; every intermediate of tenant 1's instance too.
    With c1_cache = 1 some instances read cached rows and the others draw in the same launches"""
    from eva_b200 import b200
    d, prog, params, sig, terms = _load(name, terms=True)
    pubs = [b200.generate_keys(params, seed=41 + t)[0] for t in range(3)]
    ref = {"expanded": _server(params, None, capacity=4), "seeded": _server(params, 0, capacity=4)}
    vals = [_inputs(d, pubs[t], sig, 10 + i) for i, t in enumerate(ASSIGN)]
    rq = list(zip(ASSIGN, vals))
    OPTS = ({"fuse": 1}, {"fuse": 3}, {"fuse": 3, "rotation_sums": False}, {"fuse": 1, "hoist_mod_up": False})
    for s in ref.values():
        for p in pubs:
            s.add_keys(p)
    want = {}
    for i, opts in enumerate(OPTS):
        outs = {}
        for ks, s in ref.items():
            s.set_options(**opts)
            outs[ks] = s.execute_batch(prog, rq)
        _same(d, outs["seeded"], outs["expanded"], opts)
        want[i] = outs["expanded"]
    b = ASSIGN.index(1)
    ref["expanded"].set_options(fuse=3)
    ref["expanded"].execute_batch(prog, rq)
    for H in (1, 2, 4):
        s = _server(params, H, capacity=4)
        for t, p in enumerate(pubs):
            assert s.add_keys(p) == t
        for i, opts in enumerate(OPTS):
            s.set_options(**opts)
            _same(d, s.execute_batch(prog, rq), want[i], (H, opts))
        info = s.bank_info()
        assert info["c1_cache"] == H and len(info["c1_cached"]) == min(H, 3)
        s.set_options(fuse=3)
        s.execute_batch(prog, rq)
        checked = 0
        for t in d["terms"]:
            got = s.debug_value(prog, terms[t["id"]].index, 3, b)
            w = ref["expanded"].debug_value(prog, terms[t["id"]].index, 3, b)
            assert (got is None) == (w is None), t
            if got is not None:
                assert np.array_equal(got[0], w[0]), (name, H, t)
                checked += 1
        assert checked > 0


@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_server_c1_power_of_two_paged(name):
    """power-of-two keys, 4 tenants over 2 slots, c1_cache 1 and 2, sync and async: byte-equal to the expanded inline server"""
    from eva_b200 import b200
    d, prog, params, sig = _load(name)
    pubs = [b200.generate_keys(params, seed=51 + t, rotation_keys="power_of_two")[0] for t in range(4)]
    servers = {c1: _server(params, c1, capacity=2, max_tenants=4, rotation_keys="power_of_two") for c1 in (None, 1, 2)}
    for s in servers.values():
        for t, p in enumerate(pubs):
            assert s.add_keys(p) == t
    for i, order in enumerate(([0, 1, 1, 0], [2, 3, 2], [1, 0], [0, 0, 3])):
        rq = [(t, _inputs(d, pubs[t], sig, 100 * i + j)) for j, t in enumerate(order)]
        want = servers[None].execute_batch(prog, rq)
        for c1 in (1, 2):
            _same(d, servers[c1].execute_batch(prog, rq), want, (name, order, c1))
            h = servers[c1].execute_batch_async(prog, rq)
            _same(d, servers[c1].execute_batch_result(h), want, (name, order, c1, "async"))
    for c1 in (1, 2):
        info = servers[c1].bank_info()
        assert info["evictions"] > 0 and info["c1_fills"] > c1 and info["c1_evictions"] > 0


def test_server_c1_survives_slot_eviction():
    """2 slots, 3 tenants, 2 c1 regions: [0, 1, 1] caches 1 then 0; [2] pages tenant 0's slot out and evicts tenant 1's region (the
    least recently used, lowest first); [0] pages tenant 0 back in and reads the rows cached before -- no c1 fill -- byte-equal to the
    expanded inline server"""
    from eva_b200 import b200
    d, prog, params, sig = _load("sobel")
    pubs = [b200.generate_keys(params, seed=81 + t)[0] for t in range(3)]
    servers = {c1: _server(params, c1, capacity=2, max_tenants=3) for c1 in (None, 2)}
    for s in servers.values():
        for p in pubs:
            s.add_keys(p)
    s = servers[2]
    for i, order in enumerate(([0, 1, 1], [2], [0])):
        rq = [(t, _inputs(d, pubs[t], sig, 10 * i + j)) for j, t in enumerate(order)]
        before = s.bank_info()
        _same(d, s.execute_batch(prog, rq), servers[None].execute_batch(prog, rq), order)
        after = s.bank_info()
        if order == [2]:
            assert 0 not in after["resident"] and sorted(after["c1_cached"]) == [0, 2]
        if order == [0]:
            assert after["fills"] == before["fills"] + 1 and after["c1_fills"] == before["c1_fills"]
            assert 0 in after["resident"] and 0 in after["c1_cached"]


def test_server_c1_remove_and_reuse_id():
    """remove_keys drops the tenant's region: a new client at the same id runs with its own keys"""
    from eva_b200 import b200
    d, prog, params, sig = _load("sobel")
    a, b = (b200.generate_keys(params, seed=s)[0] for s in (91, 92))
    servers = {c1: _server(params, c1, capacity=2) for c1 in (None, 1)}
    for s in servers.values():
        assert s.add_keys(a) == 0
    rq = [(0, _inputs(d, a, sig, 1))]
    _same(d, servers[1].execute_batch(prog, rq), servers[None].execute_batch(prog, rq), "a")
    assert servers[1].bank_info()["c1_cached"] == [0]
    for s in servers.values():
        s.remove_keys(0)
        assert s.add_keys(b) == 0
    assert servers[1].bank_info()["c1_cached"] == []
    rq = [(0, _inputs(d, b, sig, 2))]
    _same(d, servers[1].execute_batch(prog, rq), servers[None].execute_batch(prog, rq), "b")
    assert servers[1].bank_info()["c1_fills"] == 2


def test_server_c1_zero_digit_redo():
    """a digit with a zero coefficient: the redo on plain rotations resolves the c1 regions again and equals the expanded server"""
    from eva_b200 import b200
    d, prog, params, sig = _load("sobel")
    pub, _ = b200.generate_keys(params, seed=61)
    servers = {c1: _server(params, c1, capacity=2) for c1 in (None, 1)}
    for s in servers.values():
        s.add_keys(pub)
    (name_, _), = d["signature"].items()
    clean = _inputs(d, pub, sig, 4)
    for s in servers.values():
        s.execute_batch(prog, [(0, clean)])
    built = {c1: s.plans_built() for c1, s in servers.items()}
    val = _inputs(d, pub, sig, 3)
    kind, ct, scale = val.get(name_)
    ct = np.array(ct)
    orc = o.Oracle(params.poly_modulus_degree, list(params.prime_bits))
    ell = ct.shape[1]
    c1 = np.stack([orc.ntt_inv(ct[1, r], r) for r in range(ell)])
    c1[1, 7] = 0
    ct[1] = np.stack([orc.ntt_fwd(c1[r], r) for r in range(ell)])
    val.set_cipher(name_, ct, scale)
    outs = {c: s.execute_batch(prog, [(0, val)]) for c, s in servers.items()}
    _same(d, outs[1], outs[None], "zero digit")
    for c, s in servers.items():
        assert s.plans_built() == built[c] + 1, c
    assert servers[1].bank_info()["c1_fills"] == 1


def test_bank_info_counters_launches_and_errors():
    """a repeated batch fills nothing; a region is a slot's size; c1_cache = H issues the c1_cache=0 server's launches plus one per
    fill; the error cases name c1_cache and the option it conflicts with"""
    from eva_b200 import b200
    d, prog, params, sig = _load("sobel")
    pubs = [b200.generate_keys(params, seed=71 + t)[0] for t in range(3)]
    servers = {c1: _server(params, c1, capacity=3) for c1 in (0, 2)}
    for s in servers.values():
        for p in pubs:
            s.add_keys(p)
    rq = [(t, _inputs(d, pubs[t], sig, i)) for i, t in enumerate([2, 0, 2, 1])]
    base = {c1: s.launch_count() for c1, s in servers.items()}
    for _ in range(3):
        _same(d, servers[2].execute_batch(prog, rq), servers[0].execute_batch(prog, rq), "repeat")
    info = servers[2].bank_info()
    assert info["c1_fills"] == 2 and info["c1_evictions"] == 0 and sorted(info["c1_cached"]) == [0, 2]
    assert info["c1_cache_bytes"] == 2 * info["tenant_bytes"] and info["bank_bytes"] == 3 * info["tenant_bytes"]
    zero = servers[0].bank_info()
    assert zero["c1_cache"] == 0 and zero["c1_cache_bytes"] == 0 and zero["c1_fills"] == 0 and zero["c1_cached"] == []
    assert servers[2].launch_count() - base[2] == servers[0].launch_count() - base[0] + info["c1_fills"]
    with pytest.raises(Exception, match="c1_cache.*key_storage"):
        b200.B200Server(params, capacity=2, hoist_constants="inline", c1_cache=1)
    with pytest.raises(Exception, match="c1_cache.*key_storage"):
        b200.B200Server(params, capacity=2, c1_cache=1)
    for bad in (3, -1):
        with pytest.raises(Exception, match="c1_cache.*capacity"):
            b200.B200Server(params, capacity=2, hoist_constants="inline", key_storage="seeded", c1_cache=bad)
