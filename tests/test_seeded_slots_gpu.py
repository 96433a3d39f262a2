"""Seeded key slots on the GPU: B200Server(hoist_constants="inline", key_storage="seeded") keeps each key's c0 rows and seed and
draws the uniform half inside the key-switch inner products.  Its outputs equal, byte for byte, those of an expanded inline server
and of every tenant's own B200Public -- Sobel and Harris with 3 tenants, fuse 1 and 3, the rotation-sum, hoisted and plain
rotation paths, power-of-two keys, paging and the zero-digit redo -- and the bank sizes and the error cases are as documented."""
import ctypes as C

import numpy as np
import pytest

import parity_cases as pc
from backends import _elt
from oracle import oracle as o
from test_compressed_keys import np_expand, seeds_for
from test_rotation_wsum import WSUM_VALUES, WsumGpuBackend, _ptrs

pytestmark = pytest.mark.gpu


# ---- the C-ABI: evab_set_key_seeded against expanded keys, with and without a key-bank table

class SeededGpu(WsumGpuBackend):
    """every key of a case in four device forms: expanded [k-1][2][k][N] and seeded image (c0 rows, then the seed padded to 64
    bytes), each alone ("flat") and as region 1 of a two-region bank whose region 0 holds a decoy key (evab_set_key_bank with a
    one-instance table selecting region 1).  The expanded key's c1 rows are np_expand of its seed, so both forms are the same key"""

    def __init__(self, orc, names, salt):
        super().__init__(orc.N, orc.primes)
        N, k = orc.N, orc.k
        self.orc, self.k = orc, k
        self.kw, self.sw = (k - 1) * 2 * k * N, (k - 1) * k * N + 8
        assert self.lib.evab_seeded_key_bytes(self.h) == 8 * self.sw
        self.full, self.dev = {}, {}
        seeds = seeds_for(2 * len(names), salt)
        for i, name in enumerate(names):
            K = orc.relin_key() if name is None else orc.galois_key(name)
            forms = []
            for sd, c0 in ((seeds[2 * i], K[:, 0]), (seeds[2 * i + 1], K[:, 0, :, ::-1])):   # the key, then its decoy
                F = np.empty_like(K)
                F[:, 0] = c0
                F[:, 1] = np_expand(sd, N, orc.primes)[0]
                img = np.zeros(self.sw, dtype=np.uint64)
                img[:self.sw - 8] = F[:, 0].ravel()
                img[self.sw - 8:self.sw - 4] = np.frombuffer(sd, dtype=np.uint64)
                forms.append((F, img))
            (F, img), (D, dimg) = forms
            self.full[name] = F
            self.dev[name] = {("expanded", False): self._up(F), ("seeded", False): self._up(img),
                              ("expanded", True): self._up(np.concatenate([D.ravel(), F.ravel()])),
                              ("seeded", True): self._up(np.concatenate([dimg, img]))}
        self.table = self._up(np.array([1], dtype=np.uint64))   # int32 [1] = region 1 (little endian)
        self.elts = [e for e in names if e is not None]
        self.ind = {}
        for e in self.elts:
            self._chk(self.lib.evab_galois_prepare(self.h, C.c_uint64(e)))
            d = self._alloc(self.lib.evab_hoist_indicators_bytes(self.h, 1))
            self._chk(self.lib.evab_hoist_indicators(self.h, 1, (C.c_uint64 * 1)(e), d, None))
            self.ind[e] = d

    def modes(self, fn):
        """fn(key_of) under the four forms; returns {(storage, bank): output}.  The hoisted calls take inline constants in every form"""
        lib, out = self.lib, {}
        for storage in ("expanded", "seeded"):
            for bank in (False, True):
                key_of = lambda name: self.dev[name][(storage, bank)]
                self._chk(lib.evab_set_key_bank(self.table if bank else None, C.c_size_t(self.sw if storage == "seeded" else self.kw) if bank else C.c_size_t(0)))
                self._chk(lib.evab_set_hoist_inline(1))
                self._chk(lib.evab_set_key_seeded(1 if storage == "seeded" else 0))
                try:
                    out[(storage, bank)] = fn(key_of)
                finally:
                    lib.evab_set_key_seeded(0)
                    lib.evab_set_hoist_inline(0)
                    lib.evab_set_key_bank(None, C.c_size_t(0))
        return out

    def prepare(self, a):
        ell = a.shape[1]
        da, that, ext, zf = self._up(a), self._alloc(ell * self.N * 8), self._alloc(self.lib.evab_rotate_modup_ext_bytes(self.h, ell)), self._alloc(8)
        self._chk(self.lib.evab_memset_zero(self.h, zf, 8, None))
        self._chk(self.lib.evab_rotate_modup_prepare(self.h, ell, that, ext, da, zf, None))
        self._chk(self.lib.evab_rotate_modup_scale_c0(self.h, ell, ext, da, None))
        assert self._down(zf, (1,))[0] == 0
        return da, ext, [that, zf]

    def relinearize(self, a):
        ell = a.shape[1]
        da, do, dw = self._up(a), self._alloc(2 * ell * self.N * 8), self._alloc(self.lib.evab_keyswitch_work_bytes(self.h, ell))

        def fn(key):
            self._chk(self.lib.evab_relinearize(self.h, ell, do, da, key(None), dw, None))
            return self._down(do, (2, ell, self.N))
        r = self.modes(fn)
        self._free(da, do, dw)
        return r

    def rotate(self, a, e):
        ell = a.shape[1]
        da, do, dw = self._up(a), self._alloc(2 * ell * self.N * 8), self._alloc(self.lib.evab_keyswitch_work_bytes(self.h, ell))
        dh = self._alloc(ell * self.N * 8)
        self._chk(self.lib.evab_rotate_prepare(self.h, ell, dh, da, None))

        def fn(key):
            self._chk(self.lib.evab_rotate(self.h, ell, do, da, C.c_uint64(e), key(e), dw, None))
            plain = self._down(do, (2, ell, self.N))
            self._chk(self.lib.evab_rotate_prepared(self.h, ell, do, da, dh, C.c_uint64(e), key(e), dw, None))
            return plain, self._down(do, (2, ell, self.N))
        r = self.modes(fn)
        self._free(da, do, dw, dh)
        return r

    def modup_prepared(self, a, e):
        ell = a.shape[1]
        da, ext, tmp = self.prepare(a)
        work, do = self._alloc(self.lib.evab_rotate_modup_work_bytes(self.h, ell)), self._alloc(2 * ell * self.N * 8)

        def fn(key):
            self._chk(self.lib.evab_rotate_modup_prepared(self.h, ell, do, da, ext, C.c_uint64(e), key(e), self.ind[e], work, None))
            return self._down(do, (2, ell, self.N))
        r = self.modes(fn)
        self._free(da, ext, work, do, *tmp)
        return r

    def modup_many(self, a, elts):
        ell, n = a.shape[1], len(elts)
        da, ext, tmp = self.prepare(a)
        work, do = self._alloc(self.lib.evab_rotate_modup_many_work_bytes(self.h, ell, n)), self._alloc(n * 2 * ell * self.N * 8)

        def fn(key):
            self._chk(self.lib.evab_rotate_modup_many(self.h, ell, n, do, da, ext, (C.c_uint64 * n)(*elts), _ptrs([key(e) for e in elts]),
                                                      _ptrs([self.ind[e] for e in elts]), work, None))
            return self._down(do, (n, 2, ell, self.N))
        r = self.modes(fn)
        self._free(da, ext, work, do, *tmp)
        return r

    def wsum(self, a, elts, wts, taps, twts):
        ell, n, nout = a.shape[1], len(elts), len(wts)
        da, ext, tmp = self.prepare(a)
        dts = [self._up(t) for t in taps]
        dws = [[None if w is None else self._up(w) for w in ws] for ws in list(wts) + list(twts)]
        work, do = self._alloc(self.lib.evab_rotate_wsum_work_bytes(self.h, ell, n, nout)), self._alloc(nout * 2 * ell * self.N * 8)

        def fn(key):
            self._chk(self.lib.evab_rotate_wsum(self.h, ell, nout, do, da, ext, n, (C.c_uint64 * n)(*elts), _ptrs([key(e) for e in elts]),
                                                _ptrs([self.ind[e] for e in elts]), _ptrs([w for ws in dws[:nout] for w in ws]), len(taps),
                                                _ptrs(dts), _ptrs([w for ws in dws[nout:] for w in ws]), work, None))
            return self._down(do, (nout, 2, ell, self.N))
        r = self.modes(fn)
        self._free(da, ext, work, do, *dts, *[w for ws in dws for w in ws if w is not None], *tmp)
        return r


def _all_equal(r, what):
    """every form equals the expanded key without a bank, word for word"""
    want = r[("expanded", False)]
    for form, got in r.items():
        if isinstance(want, tuple):
            for g, w in zip(got, want):
                pc.eq(g, w)
        else:
            pc.eq(got, want)
    return want


def _cabi_seeded_case(N, bits, steps, levels=None, salt=0):
    orc = o.Oracle(N, list(bits)).keygen(3)
    elts = [_elt(N, s) for s in steps]
    be = SeededGpu(orc, [None] + elts, salt + N + len(bits))
    rng = np.random.default_rng(9)
    for ell in (levels or range(1, orc.k)):
        a3 = pc.rand_ct(orc, 3, ell, 20 + ell)
        _all_equal(be.relinearize(a3), ("relinearize", ell))
        a = pc.rand_ct(orc, 2, ell, 40 + ell)
        plain, prepared = _all_equal(be.rotate(a, elts[0]), ("rotate", ell))
        pc.eq(prepared, plain)
        hoisted = _all_equal(be.modup_prepared(a, elts[0]), ("rotate_modup_prepared", ell))
        pc.eq(hoisted, plain)
        many = _all_equal(be.modup_many(a, elts), ("rotate_modup_many", ell))
        pc.eq(many[0], plain)
        enc = lambda v: orc.encode(np.array([v]), 2.0 ** 30, ell)
        y = pc.rand_ct(orc, 2, ell, 80 + ell)
        for nout in range(1, 5):
            wts = [[None if rng.random() < 0.2 else enc(WSUM_VALUES[rng.integers(len(WSUM_VALUES))]) for _ in elts] for _ in range(nout)]
            twts = [[enc(-1.0 - oi), None if oi % 2 else enc(0.5)] for oi in range(nout)]
            _all_equal(be.wsum(a, elts, wts, [a, y], twts), ("rotate_wsum", ell, nout))
        if ell == orc.k - 1:   # the expanded key switch is the oracle's with the same key
            pc.eq(plain, orc.rotate(a, steps[0], be.full[elts[0]]))
            pc.eq(_all_equal(be.relinearize(a3), "relin"), orc.relinearize(a3, be.full[None]))
    return be


def test_cabi_seeded_sobel_shape():
    """N = 16384 on Sobel's 5 x 60-bit chain, ell = 1 .. 4: every seeded call equals the expanded one, with and without a bank"""
    _cabi_seeded_case(16384, [60] * 5, [1, 64, 130])


def test_cabi_seeded_mixed_chain():
    """a mixed 60/50/40-bit chain at N = 4096: the draw with primes of every size, another tile count per row"""
    _cabi_seeded_case(4096, [60, 50, 40, 50, 60], [1, -3, 7])


def test_cabi_seeded_deep_chain():
    """14 primes at N = 4096: at ell = 13 the 256-thread tiles of k_ks_inner and k_rot_many take 52 KB of shared memory, past the
    48 KB default"""
    _cabi_seeded_case(4096, [60] + [50] * 12 + [60], [1, -3], levels=[1, 12, 13], salt=5)


def test_cabi_seeded_refusals():
    orc = o.Oracle(4096, [60, 60, 60]).keygen(4)
    e = _elt(4096, 1)
    be = SeededGpu(orc, [None, e], 17)
    lib, ell = be.lib, 1
    a = pc.rand_ct(orc, 2, ell, 3)
    da, ext, tmp = be.prepare(a)
    key = be.dev[e][("seeded", False)]
    wt = be._up(np.zeros((ell + 1, 4096), dtype=np.uint64))
    work, do = be._alloc(lib.evab_lazy_rotsum_work_bytes(be.h, ell, 1)), be._alloc(2 * ell * 4096 * 8)
    cadd, ctmp = be._alloc(lib.evab_hoist_const_bytes(be.h, ell)), be._alloc((ell + 1) * 4096 * 8)
    mwork = be._alloc(lib.evab_rotate_modup_work_bytes(be.h, ell))
    lib.evab_set_key_seeded(1)
    try:
        lib.evab_set_hoist_inline(1)
        rc = lib.evab_lazy_rotsum(be.h, ell, 1, do, da, ext, 1, (C.c_uint64 * 1)(e), _ptrs([key]), _ptrs([be.ind[e]]), _ptrs([wt]), work, None)
        assert rc != 0 and b"lazy_rotsum" in lib.evab_last_error()
        lib.evab_set_hoist_inline(0)
        rc = lib.evab_rotate_hoist_const(be.h, ell, C.c_uint64(e), key, cadd, ctmp, None)
        assert rc != 0 and b"evab_set_key_seeded" in lib.evab_last_error()
        rc = lib.evab_rotate_modup_prepared(be.h, ell, do, da, ext, C.c_uint64(e), key, cadd, mwork, None)
        assert rc != 0 and b"inline hoist constants" in lib.evab_last_error()
    finally:
        lib.evab_set_key_seeded(0)
        lib.evab_set_hoist_inline(0)
    be._free(da, ext, wt, work, do, cadd, ctmp, mwork, *tmp)


# ---- B200Server(hoist_constants="inline", key_storage="seeded")

ASSIGN = [0, 1, 2, 1, 0, 2]


def _load(name, terms=False):
    from eva_b200 import program_io as gl
    d = gl.load_json(name)
    prog, params, sig, tm = gl.build_program(d)
    return (d, prog, params, sig, tm) if terms else (d, prog, params, sig)


def _servers(params, **kw):
    from eva_b200 import b200
    return {ks: b200.B200Server(params, hoist_constants="inline", key_storage=ks, **kw) for ks in ("expanded", "seeded")}


def _inputs(d, pub, sig, seed):
    rng = np.random.default_rng(seed)
    return pub.encrypt({nm: list(rng.uniform(0, 0.2, d["vec_size"])) for nm in d["signature"]}, sig)


def _same(d, a, b, what):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        for oname in d["outputs"]:
            assert np.array_equal(x.get(oname)[1], y.get(oname)[1]), (what, oname)


@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_server_seeded_bit_exact(name):
    """3 tenants in one batch: fuse 1 and 3, without rotation sums (the batched hoisted rotations) and without the shared mod-up (plain
    rotations): the seeded server equals the expanded inline server and each tenant's own context, and every intermediate of one
    tenant's instance equals the expanded server's"""
    from eva_b200 import b200
    d, prog, params, sig, terms = _load(name, terms=True)
    servers = _servers(params, capacity=4)
    pubs = [b200.generate_keys(params, seed=41 + t)[0] for t in range(3)]
    for s in servers.values():
        for t, p in enumerate(pubs):
            assert s.add_keys(p) == t
    info = servers["seeded"].bank_info()
    assert info["key_storage"] == "seeded" and info["compressed_tenants"] == info["tenants"] == 3
    vals = [_inputs(d, pubs[t], sig, 10 + i) for i, t in enumerate(ASSIGN)]
    for opts in ({"fuse": 1}, {"fuse": 3}, {"fuse": 3, "rotation_sums": False}, {"fuse": 1, "hoist_mod_up": False}):
        outs = {}
        for ks, s in servers.items():
            s.set_options(**opts)
            outs[ks] = s.execute_batch(prog, list(zip(ASSIGN, vals)))
        _same(d, outs["seeded"], outs["expanded"], ("expanded", opts))
        for t in range(3):
            mine = [i for i, a in enumerate(ASSIGN) if a == t]
            pubs[t].set_options(**opts)
            _same(d, [outs["seeded"][i] for i in mine], pubs[t].execute_batch(prog, [vals[i] for i in mine]), ("public", opts, t))
    # every intermediate of tenant 1's instance equals the expanded server's
    b = ASSIGN.index(1)
    for s in servers.values():
        s.set_options(fuse=3)
        s.execute_batch(prog, list(zip(ASSIGN, vals)))
    checked = 0
    for t in d["terms"]:
        got = servers["seeded"].debug_value(prog, terms[t["id"]].index, 3, b)
        want = servers["expanded"].debug_value(prog, terms[t["id"]].index, 3, b)
        assert (got is None) == (want is None), t
        if got is not None:
            assert np.array_equal(got[0], want[0]), (name, t)
            checked += 1
    assert checked > 0


@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_server_seeded_power_of_two_paged(name):
    """power-of-two keys, 4 tenants over 2 slots (evictions and refills between submits), sync and async: the seeded server's outputs
    equal the expanded inline server's, byte for byte, and fills are counted"""
    from eva_b200 import b200
    d, prog, params, sig = _load(name)
    servers = _servers(params, capacity=2, max_tenants=4, rotation_keys="power_of_two")
    pubs = [b200.generate_keys(params, seed=51 + t, rotation_keys="power_of_two")[0] for t in range(4)]
    for s in servers.values():
        for t, p in enumerate(pubs):
            assert s.add_keys(p) == t
        assert s.bank_info()["compressed_tenants"] == 4
    for i, order in enumerate(([0, 1, 1, 0], [2, 3, 2], [1, 0])):
        rq = [(t, _inputs(d, pubs[t], sig, 100 * i + j)) for j, t in enumerate(order)]
        outs = {ks: s.execute_batch(prog, rq) for ks, s in servers.items()}
        _same(d, outs["seeded"], outs["expanded"], (name, order))
        h = servers["seeded"].execute_batch_async(prog, rq)
        _same(d, servers["seeded"].execute_batch_result(h), outs["expanded"], (name, order, "async"))
    info = servers["seeded"].bank_info()
    assert info["evictions"] > 0 and info["fills"] > 4


def test_server_seeded_zero_digit_redo():
    """an instance whose digit has a zero coefficient takes the redo on plain rotations (evab_rotate_prepared with seeded keys): the
    seeded server equals the expanded inline server"""
    from eva_b200 import b200
    d, prog, params, sig = _load("sobel")
    servers = _servers(params, capacity=2)
    pub, _ = b200.generate_keys(params, seed=61)
    for s in servers.values():
        s.add_keys(pub)
    (name_, info), = d["signature"].items()
    clean = _inputs(d, pub, sig, 4)
    for s in servers.values():   # builds the plans that share their mod-up
        s.execute_batch(prog, [(0, clean)])
    built = {ks: s.plans_built() for ks, s in servers.items()}
    val = _inputs(d, pub, sig, 3)
    kind, ct, scale = val.get(name_)
    assert kind == "cipher"
    ct = np.array(ct)
    from oracle import oracle as o
    orc = o.Oracle(params.poly_modulus_degree, list(params.prime_bits))
    ell = ct.shape[1]
    c1 = np.stack([orc.ntt_inv(ct[1, r], r) for r in range(ell)])
    c1[1, 7] = 0
    ct[1] = np.stack([orc.ntt_fwd(c1[r], r) for r in range(ell)])
    val.set_cipher(name_, ct, scale)
    outs = {ks: s.execute_batch(prog, [(0, val)]) for ks, s in servers.items()}
    _same(d, outs["seeded"], outs["expanded"], "zero digit")
    # the flag was raised and the batch redone on a plan without the shared mod-up (plain rotations, evab_rotate_prepared)
    for ks, s in servers.items():
        assert s.plans_built() == built[ks] + 1, ks


def test_bank_info_sizes_and_errors():
    """seeded slots are half the inline ones plus 64 bytes per key, at Sobel's shape with both key sets; the error cases"""
    from eva_b200 import b200
    d, prog, params, sig = _load("sobel")
    want = {"program": 52428800, "power_of_two": 26214400}
    for keys, inline_bytes in want.items():
        infos = {ks: s.bank_info() for ks, s in _servers(params, capacity=2, rotation_keys=keys).items()}
        nkeys = 1 + len(infos["seeded"]["galois_elements"])
        assert infos["expanded"]["tenant_bytes"] == inline_bytes and infos["expanded"]["key_storage"] == "expanded"
        seeded = infos["seeded"]
        assert seeded["tenant_bytes"] == inline_bytes // 2 + 64 * nkeys, (keys, seeded)
        assert seeded["key_bytes_per_tenant"] == seeded["tenant_bytes"] and seeded["bank_bytes"] == 2 * seeded["tenant_bytes"]
        assert seeded["hoist_const_bytes_per_tenant"] == 0 and seeded["fills"] == 0
    for bad in ({"hoist_constants": "stored", "key_storage": "seeded"}, {"hoist_constants": "inline", "key_storage": "compact"}):
        with pytest.raises(Exception, match="key_storage.*hoist_constants"):
            b200.B200Server(params, capacity=2, **bad)
    s = b200.B200Server(params, capacity=2, hoist_constants="inline", key_storage="seeded")
    pub, _ = b200.generate_keys(params, seed=71)
    k = len(params.prime_bits)
    N = params.poly_modulus_degree
    relin = np.zeros((k - 1, 2, k, N), dtype=np.uint64)
    gal = {e: relin for e in s.bank_info()["galois_elements"]}
    with pytest.raises(Exception, match="key_storage"):
        s.add_raw_keys(relin, gal)
    # a context without seeds (built from raw keys) travels in full: refused as well
    raw = b200.context_from_raw_keys(N, s.primes(), relin, gal)
    with pytest.raises(Exception, match="key_storage"):
        s.add_keys(raw)
    assert s.add_keys(pub) == 0 and s.bank_info()["fills"] == 1
    s.set_options(approx_hoist=True)
    with pytest.raises(Exception, match="approx_hoist"):
        s.execute_batch(prog, [(0, _inputs(d, pub, sig, 1))])
