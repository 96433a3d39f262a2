"""Inline hoist constants on the GPU: the C-ABI ops with evab_set_hoist_inline against the stored constants and the oracle, and
B200Server(hoist_constants="inline") against a stored server, each tenant's own B200Public and the oracle, byte for byte."""
import ctypes as C

import numpy as np
import pytest

import parity_cases as pc
from backends import _elt
from oracle import oracle as o
from test_rotation_wsum import WSUM_VALUES, WsumGpuBackend, _ptrs
from test_tenants import ASSIGN, PERMUTED, Fixture, _own_context

pytestmark = pytest.mark.gpu


class InlineGpu(WsumGpuBackend):
    """the hoisted rotation ops of the C-ABI with one Galois key per element shared by all instances, run twice: with the stored
    constant (evab_rotate_hoist_const) and with the element's indicator rows under evab_set_hoist_inline"""

    def elt(self, s):
        e = _elt(self.N, s)
        if e not in self._prepared:
            self._chk(self.lib.evab_galois_prepare(self.h, C.c_uint64(e)))
            self._prepared.add(e)
        return e

    def indicators(self, elts):
        lib = self.lib
        d = self._alloc(lib.evab_hoist_indicators_bytes(self.h, len(elts)))
        self._chk(lib.evab_hoist_indicators(self.h, len(elts), (C.c_uint64 * len(elts))(*elts), d, None))
        return d

    def operands(self, steps, gks, ell):
        """per rotation: element, device key, stored constant, indicator rows"""
        elts = [self.elt(s) for s in steps]
        keys, cadds = [self._up(g) for g in gks], []
        for e, dk in zip(elts, keys):
            cadd, tmp = self._alloc(self.lib.evab_hoist_const_bytes(self.h, ell)), self._alloc((ell + 1) * self.N * 8)
            self._chk(self.lib.evab_rotate_hoist_const(self.h, ell, C.c_uint64(e), dk, cadd, tmp, None))
            self._free(tmp)
            cadds.append(cadd)
        inds = [self.indicators([e]) for e in elts]
        return elts, keys, cadds, inds

    def prepare(self, a):
        ell = a.shape[1]
        da, that, ext, zf = self._up(a), self._alloc(ell * self.N * 8), self._alloc(self.lib.evab_rotate_modup_ext_bytes(self.h, ell)), self._alloc(8)
        self._chk(self.lib.evab_memset_zero(self.h, zf, 8, None))
        self._chk(self.lib.evab_rotate_modup_prepare(self.h, ell, that, ext, da, zf, None))
        self._chk(self.lib.evab_rotate_modup_scale_c0(self.h, ell, ext, da, None))
        assert self._down(zf, (1,))[0] == 0
        return da, ext, [that, zf]

    def both(self, fn):
        """fn(constants) with the stored constants, then with the indicator rows under evab_set_hoist_inline"""
        want = fn(False)
        self._chk(self.lib.evab_set_hoist_inline(1))
        try:
            got = fn(True)
        finally:
            self._chk(self.lib.evab_set_hoist_inline(0))
        return got, want

    def modup_prepared(self, a, s, gk):
        ell = a.shape[1]
        da, ext, tmp = self.prepare(a)
        (e,), (dk,), (cadd,), (ind,) = self.operands([s], [gk], ell)
        work, do = self._alloc(self.lib.evab_rotate_modup_work_bytes(self.h, ell)), self._alloc(2 * ell * self.N * 8)

        def fn(inl):
            self._chk(self.lib.evab_rotate_modup_prepared(self.h, ell, do, da, ext, C.c_uint64(e), dk, ind if inl else cadd, work, None))
            return self._down(do, (2, ell, self.N))
        r = self.both(fn)
        self._free(da, ext, dk, cadd, ind, work, do, *tmp)
        return r

    def modup_many(self, a, steps, gks):
        ell, n = a.shape[1], len(steps)
        da, ext, tmp = self.prepare(a)
        elts, keys, cadds, inds = self.operands(steps, gks, ell)
        work, do = self._alloc(self.lib.evab_rotate_modup_many_work_bytes(self.h, ell, n)), self._alloc(n * 2 * ell * self.N * 8)

        def fn(inl):
            self._chk(self.lib.evab_rotate_modup_many(self.h, ell, n, do, da, ext, (C.c_uint64 * n)(*elts), _ptrs(keys), _ptrs(inds if inl else cadds),
                                                      work, None))
            return self._down(do, (n, 2, ell, self.N))
        r = self.both(fn)
        self._free(da, ext, work, do, *keys, *cadds, *inds, *tmp)
        return r

    def wsum(self, a, steps, gks, wts, taps, twts):
        ell, n, nout = a.shape[1], len(steps), len(wts)
        da, ext, tmp = self.prepare(a)
        elts, keys, cadds, inds = self.operands(steps, gks, ell)
        dts = [self._up(t) for t in taps]
        dws = [[None if w is None else self._up(w) for w in ws] for ws in list(wts) + list(twts)]
        work, do = self._alloc(self.lib.evab_rotate_wsum_work_bytes(self.h, ell, n, nout)), self._alloc(nout * 2 * ell * self.N * 8)

        def fn(inl):
            self._chk(self.lib.evab_rotate_wsum(self.h, ell, nout, do, da, ext, n, (C.c_uint64 * n)(*elts), _ptrs(keys), _ptrs(inds if inl else cadds),
                                                _ptrs([w for ws in dws[:nout] for w in ws]), len(taps), _ptrs(dts),
                                                _ptrs([w for ws in dws[nout:] for w in ws]), work, None))
            return self._down(do, (nout, 2, ell, self.N))
        r = self.both(fn)
        self._free(da, ext, work, do, *keys, *cadds, *inds, *dts, *[w for ws in dws for w in ws if w is not None], *tmp)
        return r


def _gk(orc, s):
    return orc.galois_key(o.galois_elt_from_step(orc.N, s))


def _cabi_case(N, bits, steps):
    orc = pc.get_oracle(N, bits)
    be = InlineGpu(N, orc.primes)
    rng = np.random.default_rng(5)
    for ell in range(1, orc.k):
        a = pc.rand_ct(orc, 2, ell, 40 + ell)
        rots = [orc.rotate(a, s, _gk(orc, s)) for s in steps]
        got, want = be.modup_prepared(a, steps[0], _gk(orc, steps[0]))
        pc.eq(got, want); pc.eq(got, rots[0])
        got, want = be.modup_many(a, steps, [_gk(orc, s) for s in steps])
        pc.eq(got, want)
        for i in range(len(steps)):
            pc.eq(got[i], rots[i])
        enc = lambda v: orc.encode(np.array([v]), 2.0 ** 30, ell)
        nout = 1 + ell % 4
        wts = [[None if rng.random() < 0.2 else enc(WSUM_VALUES[rng.integers(len(WSUM_VALUES))]) for _ in steps] for _ in range(nout)]
        y = pc.rand_ct(orc, 2, ell, 80 + ell)
        twts = [[enc(-1.0 - oi), None if oi % 2 else enc(0.5)] for oi in range(nout)]
        got, want = be.wsum(a, steps, [_gk(orc, s) for s in steps], wts, [a, y], twts)
        pc.eq(got, want)
        for oi in range(nout):
            acc = None
            for c_, w in list(zip(rots, wts[oi])) + list(zip([a, y], twts[oi])):
                if w is not None:
                    term = orc.mul_plain(c_, w)
                    acc = term if acc is None else orc.add(acc, term)
            pc.eq(got[oi], acc)
    return orc, be


def test_cabi_inline_sobel_shape():
    """N = 16384 on Sobel's chain, ell = 1 .. 4: inline == stored == the oracle for the three ops"""
    _cabi_case(16384, [60] * 5, [1, 64, 130])


def test_cabi_inline_mixed_chain():
    """a mixed 60/50/40-bit chain at N = 4096 (q_J mod m is a real reduction), and the indicator rows are the factor of
    evab_rotate_hoist_const_levels' constants: cadd[c][m] = ind[m] (.) sum_J (q_J mod m) K[J][c][m] for every level"""
    orc, be = _cabi_case(4096, [60, 50, 40, 50, 60], [1, -3, 7])
    N, k, primes = orc.N, orc.k, [int(p) for p in orc.primes]
    elts = [be.elt(s) for s in (1, -3)]
    keys = np.stack([_gk(orc, s) for s in (1, -3)])
    dk, dind = be._up(keys), be.indicators(elts)
    per = be.lib.evab_hoist_const_levels_bytes(be.h) // 8
    dout, dtmp = be._alloc(2 * per * 8), be._alloc(be.lib.evab_rotate_hoist_const_levels_work_bytes(be.h, 2))
    be._chk(be.lib.evab_rotate_hoist_const_levels(be.h, 2, (C.c_uint64 * 2)(*elts), dk, dout, dtmp, None))
    consts, ind = be._down(dout, (2, per)), be._down(dind, (2, k, N))
    for g in range(2):
        off = 0
        for ell in range(1, k):
            blk = consts[g, off:off + 2 * (ell + 1) * N].reshape(2, ell + 1, N)
            off += 2 * (ell + 1) * N
            for mi in range(ell + 1):
                m = mi if mi < ell else k - 1
                for c in range(2):
                    s = sum((primes[J] % primes[m]) * keys[g, J, c, m].astype(object) for J in range(ell)) % primes[m]
                    assert np.array_equal(blk[c, mi], ((s * ind[g, m].astype(object)) % primes[m]).astype(np.uint64)), (g, ell, mi, c)
    be._free(dk, dind, dout, dtmp)


def test_cabi_lazy_rotsum_refuses_inline():
    orc = pc.get_oracle(4096, [60, 60, 60])
    be = InlineGpu(4096, orc.primes)
    ell = 1
    da, ext, tmp = be.prepare(pc.rand_ct(orc, 2, ell, 3))
    (e,), (dk,), _, (ind,) = be.operands([1], [_gk(orc, 1)], ell)
    wt = be._up(np.zeros((ell + 1, 4096), dtype=np.uint64))
    work, do = be._alloc(be.lib.evab_lazy_rotsum_work_bytes(be.h, ell, 1)), be._alloc(2 * ell * 4096 * 8)
    be._chk(be.lib.evab_set_hoist_inline(1))
    try:
        rc = be.lib.evab_lazy_rotsum(be.h, ell, 1, do, da, ext, 1, (C.c_uint64 * 1)(e), _ptrs([dk]), _ptrs([ind]), _ptrs([wt]), work, None)
    finally:
        be._chk(be.lib.evab_set_hoist_inline(0))
    assert rc != 0 and b"approx_hoist" in be.lib.evab_last_error()


# ---- B200Server(hoist_constants="inline")

class InlineFixture(Fixture):
    """test_tenants.Fixture (3 tenants with oracle keys, 6 instances) on a server with the given options, plus a stored twin"""

    def __init__(self, name, capacity=4, **server):
        from eva_b200 import b200
        real = b200.B200Server
        try:   # Fixture builds its server as B200Server(params, capacity=...): give it the options under test
            b200.B200Server = lambda params, capacity: real(params, capacity=capacity, **server)
            super().__init__(name, capacity=capacity)
        finally:
            b200.B200Server = real
        self.stored = real(self.params, capacity=capacity, **dict(server, hoist_constants="stored"))
        for rk_gks in self.keys:
            self.stored.add_raw_keys(*rk_gks)

    def same(self, a, b, what):
        for x, y in zip(a, b):
            for oname in self.d["outputs"]:
                assert np.array_equal(x.get(oname)[1], y.get(oname)[1]), (what, oname)


@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_server_inline_bit_exact(name):
    """3 tenants in one batch, fuse 1 and a batched plan (fuse 3): every output equals the stored server's, the tenant's own
    B200Public and the oracle; every intermediate of tenant 1's instance equals the oracle runner"""
    f = InlineFixture(name, hoist_constants="inline")
    assert f.server.bank_info()["hoist_constants"] == "inline"
    pubs = [_own_context(f, t) for t in range(3)]
    for fuse in (1, 3):
        outs = f.run(ASSIGN, fuse=fuse)
        f.stored.set_options(fuse=fuse)
        f.same(outs, f.stored.execute_batch(f.prog, list(zip(ASSIGN, f.vals))), ("stored", fuse))
        f.check(outs, ASSIGN, ("oracle", fuse))
        for t in range(3):
            mine = [i for i, a in enumerate(ASSIGN) if a == t]
            pubs[t].set_options(fuse=fuse)
            f.same([outs[i] for i in mine], pubs[t].execute_batch(f.prog, [f.vals[i] for i in mine]), ("public", fuse, t))
    f.check(f.run(PERMUTED), PERMUTED, "permuted")
    f.drop_plans()
    f.check(f.run(ASSIGN, fuse=3, fuse_sums=False), ASSIGN, "materialised")
    b = ASSIGN.index(1)
    for t in f.d["terms"]:
        want = f.want(b, 1)[t["id"]]
        if want[0] == "raw":
            continue
        got = f.server.debug_value(f.prog, f.terms[t["id"]].index, 3, b)
        w = want[1] if want[0] == "cipher" else want[1][None]
        assert got is not None and np.array_equal(got[0], w), (name, t)


@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_server_inline_power_of_two_compressed_paged(name):
    """power-of-two keys, compressed tenants and paging (4 tenants over 2 slots, evictions and refills between submits): the
    inline server's outputs equal the stored server's, byte for byte"""
    from eva_b200 import b200, program_io as gl
    d = gl.load_json(name)
    prog, params, sig, _ = gl.build_program(d)
    servers = {h: b200.B200Server(params, capacity=2, max_tenants=4, rotation_keys="power_of_two", hoist_constants=h) for h in ("stored", "inline")}
    pubs = [b200.generate_keys(params, seed=31 + t, rotation_keys="power_of_two")[0] for t in range(4)]
    for s in servers.values():
        for t, p in enumerate(pubs):
            assert s.add_keys(p) == t
        assert s.bank_info()["compressed_tenants"] == 4
    rng = np.random.default_rng(2)
    enc = lambda t: (t, pubs[t].encrypt({nm: list(rng.uniform(0, 0.2, d["vec_size"])) for nm in d["signature"]}, sig))
    # at most 2 distinct tenants per batch (2 slots): every batch after the first evicts and refills
    for order in ([enc(t) for t in (0, 1, 1, 0)], [enc(t) for t in (2, 3, 2)], [enc(t) for t in (1, 0)]):
        outs = {h: s.execute_batch(prog, order) for h, s in servers.items()}
        for x, y in zip(outs["inline"], outs["stored"]):
            for oname in d["outputs"]:
                assert np.array_equal(x.get(oname)[1], y.get(oname)[1]), (name, oname)
    info = servers["inline"].bank_info()
    assert info["evictions"] > 0 and info["fills"] > 4 and info["hoist_const_bytes_per_tenant"] == 0


def test_server_inline_zero_digit_falls_back():
    """an instance with a zero digit coefficient on an inline server: the redo on the exact path gives the stored server's and the
    oracle's outputs"""
    f = InlineFixture("sobel", hoist_constants="inline")
    (name_, info), = f.d["signature"].items()
    i = ASSIGN.index(1)
    orc = f.orcs[1]
    ell = orc.k - 1 - info["level"]
    ct = f.ins[i][name_][1].copy()
    c1 = np.stack([orc.ntt_inv(ct[1, r], r) for r in range(ell)])
    c1[1, 7] = 0
    ct[1] = np.stack([orc.ntt_fwd(c1[r], r) for r in range(ell)])
    f.vals[i].set_cipher(name_, ct, 2.0 ** info["scale"])
    f.ins[i] = {name_: ("cipher", ct, 2.0 ** info["scale"])}
    outs = f.run(ASSIGN, fuse=3)
    f.check(outs, ASSIGN, "zero digit")
    f.stored.set_options(fuse=3)
    f.same(outs, f.stored.execute_batch(f.prog, list(zip(ASSIGN, f.vals))), "stored")


def test_bank_info_sizes_and_errors():
    """keys-only strides at Sobel's shape (both key sets), and the error cases"""
    from eva_b200 import b200, program_io as gl
    d = gl.load_json("sobel")
    prog, params, _, _ = gl.build_program(d)
    want = {("program", "stored"): (85458944, 33030144, 0), ("program", "inline"): (52428800, 0, 5898240),
            ("power_of_two", "stored"): (40894464, 14680064, 0), ("power_of_two", "inline"): (26214400, 0, 2621440)}
    for (keys, hoist), (tenant, const, ind) in want.items():
        s = b200.B200Server(params, capacity=2, rotation_keys=keys, hoist_constants=hoist)
        info = s.bank_info()
        assert (info["tenant_bytes"], info["hoist_const_bytes_per_tenant"], info["indicator_bytes"]) == (tenant, const, ind), (keys, hoist, info)
        assert info["bank_bytes"] == 2 * tenant and info["hoist_constants"] == hoist
    with pytest.raises(Exception, match='"stored" or "inline"'):
        b200.B200Server(params, capacity=2, hoist_constants="lazy")
    f = InlineFixture("sobel", capacity=3, hoist_constants="inline")
    f.server.set_options(approx_hoist=True)
    with pytest.raises(Exception, match="approx_hoist"):
        f.server.execute_batch(f.prog, [(0, f.vals[0])])
