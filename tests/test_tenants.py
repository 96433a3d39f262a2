"""Multi-tenant execution: per-instance key selection from a key bank (evab_set_key_bank), replayed on the CPU against the oracle
with each tenant's own keys, and B200Server on the GPU against the oracle run with each instance's own keys."""
import ctypes as C

import numpy as np
import pytest

import parity_cases as pc
from backends import _elt, _p
from oracle import oracle as o
from test_rotation_wsum import WSUM_STEPS, WsumEmuBackend, case_rotation_wsum

# ---------------------------------------------------------------------------------------------------------------------------
# CPU replay: a bank of 3 tenants in one host array, laid out as B200Server's KeyBank lays it out


class _BankLib:
    """the emulator library with the key-switch entry points replaced by their key-bank replays (emub_*)"""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        if name.startswith("emu_") and hasattr(self._lib, "emub_" + name[4:]):
            return getattr(self._lib, "emub_" + name[4:])
        return getattr(self._lib, name)


class Bank:
    """relinearization key, Galois keys (sorted elements), hoist constants of every (element, ell < k) per tenant"""

    def __init__(self, be, orcs, steps):
        N, k = be.N, be.k
        self.N, self.k, self.elts = N, k, sorted({_elt(N, s) for s in steps})
        self.kw = (k - 1) * 2 * k * N
        self.cw = sum(2 * (ell + 1) * N for ell in range(1, k))
        self.stride = self.kw * (1 + len(self.elts)) + self.cw * len(self.elts)
        self.words = np.zeros((len(orcs), self.stride), dtype=np.uint64)
        self.orcs = orcs
        be.lib.emu_set_key_bank(None, C.c_size_t(0))
        for t, orc in enumerate(orcs):
            self.words[t, :self.kw] = orc.relin_key().ravel()
            for i, e in enumerate(self.elts):
                self.words[t, self.kw * (1 + i):self.kw * (2 + i)] = orc.galois_key(e).ravel()
                for ell in range(1, k):
                    tmp = np.empty((ell + 1, N), dtype=np.uint64)
                    be._chk(be.lib.emu_rotate_hoist_const(be.h, ell, C.c_uint64(e), C.c_void_p(self.ptr(self.galois_off(e), t)),
                                                          C.c_void_p(self.ptr(self.cadd_off(e, ell), t)), _p(tmp)))

    def galois_off(self, e):
        return self.kw * (1 + self.elts.index(e))

    def cadd_off(self, e, ell):
        return self.kw * (1 + len(self.elts)) + self.cw * self.elts.index(e) + sum(2 * (l_ + 1) * self.N for l_ in range(1, ell))

    def ptr(self, off, t=0):
        return self.words.ctypes.data + 8 * (t * self.stride + off)

    def view(self, off, shape):
        """tenant 0's copy as an array (what a plan passes; the kernels add the instance's tenant offset)"""
        return self.words[0, off:off + int(np.prod(shape))].reshape(shape)


class BankEmuBackend(WsumEmuBackend):
    """the parity cases' key-switch ops with every key and hoist constant read from the bank for tenant `tenant`: the keys the cases
    pass in are checked to be that tenant's and replaced by tenant 0's copies"""
    SRC, LIB = "emu_bank.cpp", "libevab_emu_bank"

    def __init__(self, N, primes):
        super().__init__(N, primes)
        self.lib = _BankLib(self.lib)
        self.bank, self.table = None, np.zeros(1, dtype=np.int32)

    def select(self, bank, t):
        self.bank, self.table[0] = bank, t
        self.lib.emu_set_key_bank(self.table.ctypes.data_as(C.c_void_p), C.c_size_t(bank.stride))

    def _gk(self, steps, gk):
        e = _elt(self.N, steps)
        off = self.bank.galois_off(e)
        assert np.array_equal(self.bank.words[self.table[0], off:off + self.bank.kw], gk.ravel())
        return self.bank.view(off, gk.shape), e

    def relinearize(self, a, rk):
        assert np.array_equal(self.bank.words[self.table[0], :self.bank.kw], rk.ravel())
        return super().relinearize(a, self.bank.view(0, rk.shape))

    def rotate(self, a, steps, gk):
        return super().rotate(a, steps, self._gk(steps, gk)[0])

    def rotate_many(self, a, steps_list, gks):
        return super().rotate_many(a, steps_list, [self._gk(s, g)[0] for s, g in zip(steps_list, gks)])

    def _prepare(self, a, scale_c0=True):
        ell = a.shape[1]
        that, ext, zflag = np.empty((ell, self.N), dtype=np.uint64), np.zeros((ell + 1, ell, self.N), dtype=np.uint64), np.zeros(1, dtype=np.uint64)
        self._chk(self.lib.emu_rotate_modup_prepare(self.h, ell, _p(that), _p(ext), _p(a), _p(zflag)))
        if scale_c0:
            self._chk(self.lib.emu_rotate_modup_scale_c0(self.h, ell, _p(ext), _p(a)))
        return ext, zflag

    def _hoisted(self, steps_list, gks, ell):
        keys = [self._gk(s, g) for s, g in zip(steps_list, gks)]
        return ((C.c_uint64 * len(keys))(*[e for _, e in keys]), (C.c_void_p * len(keys))(*[k.ctypes.data for k, _ in keys]),
                (C.c_void_p * len(keys))(*[self.bank.ptr(self.bank.cadd_off(e, ell)) for _, e in keys]))

    def rotate_many_modup(self, a, steps_list, gks):
        ell, n = a.shape[1], len(steps_list)
        ext, zflag = self._prepare(a, scale_c0=False)
        elts, keys, cadds = self._hoisted(steps_list, gks, ell)
        outs = []
        for i in range(n):
            out = np.empty((2, ell, self.N), dtype=np.uint64)
            work = np.zeros(self.lib.emu_rotate_modup_work_bytes(self.h, ell) // 8, dtype=np.uint64)
            self._chk(self.lib.emu_rotate_modup_prepared(self.h, ell, _p(out), _p(a), _p(ext), C.c_uint64(elts[i]), C.c_void_p(keys[i]),
                                                         C.c_void_p(cadds[i]), _p(work)))
            outs.append(out)
        self._chk(self.lib.emu_rotate_modup_scale_c0(self.h, ell, _p(ext), _p(a)))
        self.lib.emu_rotate_modup_many_work_bytes.restype = C.c_size_t
        work = np.zeros(self.lib.emu_rotate_modup_many_work_bytes(self.h, ell, n) // 8, dtype=np.uint64)
        many = np.empty((n, 2, ell, self.N), dtype=np.uint64)
        self._chk(self.lib.emu_rotate_modup_many(self.h, ell, n, _p(many), _p(a), _p(ext), elts, keys, cadds, _p(work)))
        self.many = [many[i] for i in range(n)]
        return outs, int(zflag[0])

    def rotate_wsum(self, a, steps_list, gks, wts, taps, twts):
        ell, n, nout = a.shape[1], len(steps_list), len(wts)
        ext, zflag = self._prepare(a)
        elts, keys, cadds = self._hoisted(steps_list, gks, ell)
        taps = [np.ascontiguousarray(t) for t in taps]
        ptr = lambda w: None if w is None else w.ctypes.data
        wl = (C.c_void_p * (nout * n))(*[ptr(w) for ws in wts for w in ws])
        tl = (C.c_void_p * max(1, len(taps)))(*[t.ctypes.data for t in taps])
        twl = (C.c_void_p * max(1, nout * len(taps)))(*[ptr(w) for ws in twts for w in ws])
        work = np.zeros(self.lib.emu_rotate_wsum_work_bytes(self.h, ell, n, nout) // 8, dtype=np.uint64)
        out = np.empty((nout, 2, ell, self.N), dtype=np.uint64)
        self._chk(self.lib.emu_rotate_wsum(self.h, ell, nout, _p(out), _p(a), _p(ext), n, elts, keys, cadds, wl, len(taps), tl, twl, _p(work)))
        return out, int(zflag[0])

    def lazy_rotsum_with(self, a, steps_list, gks, pts):
        """evab_lazy_rotsum with given plaintext weights [nout][n] ([ell+1][N] each, None: not in that sum)"""
        ell, n, nout = a.shape[1], len(steps_list), len(pts)
        ext, _ = self._prepare(a)
        elts, keys, cadds = self._hoisted(steps_list, gks, ell)
        wl = (C.c_void_p * (nout * n))(*[None if w is None else w.ctypes.data for ws in pts for w in ws])
        self.lib.emu_lazy_rotsum_work_bytes.restype = C.c_size_t
        work = np.zeros(self.lib.emu_lazy_rotsum_work_bytes(self.h, ell, nout) // 8, dtype=np.uint64)
        out = np.empty((nout, 2, ell, self.N), dtype=np.uint64)
        self._chk(self.lib.emu_lazy_rotsum(self.h, ell, nout, _p(out), _p(a), _p(ext), n, elts, keys, cadds, wl, _p(work)))
        return out


STEPS = (1, -2, 7, 64)
BANK_STEPS = STEPS + WSUM_STEPS[:4]     # the bank holds every element the cases rotate by


def test_key_bank_replay_matches_each_tenants_oracle():
    """relinearize, rotate (plain, prepared, shared mod-up one by one and batched) and the weighted rotation sums, run with the
    tenant table pointing at tenant 0, 1 and 2 of a bank of oracle keys with different seeds: each equals the oracle with that
    tenant's own keys, word for word"""
    N, bits = 1024, [60, 60, 60, 60]
    orcs = [o.Oracle(N, bits).keygen(seed) for seed in (1, 2, 3)]
    be = BankEmuBackend(N, orcs[0].primes)
    bank = Bank(be, orcs, BANK_STEPS)
    try:
        for t in (0, 1, 2, 1):
            be.select(bank, t)
            for ell in (1, 3):
                pc.case_keyswitch(be, orcs[t], ell, steps=STEPS)
            case_rotation_wsum(be, orcs[t], 2, 4, 2, seed=t)
            case_rotation_wsum(be, orcs[t], 3, 3, 1, seed=t + 5)
    finally:
        be.lib.emu_set_key_bank(None, C.c_size_t(0))


def test_key_bank_replay_lazy_rotsum():
    """approx_hoist's sums (not the reference's rounding, so no oracle bits): with the table at tenant t, the same words as the
    shared-key replay given tenant t's keys, which are graded against the oracle by the existing case; tenants differ"""
    N, bits = 1024, [60, 60, 60, 60]
    orcs = [o.Oracle(N, bits).keygen(seed) for seed in (1, 2, 3)]
    be = BankEmuBackend(N, orcs[0].primes)
    plain = WsumEmuBackend(N, orcs[0].primes)
    bank = Bank(be, orcs, BANK_STEPS)
    rng = np.random.default_rng(8)
    ell = 2
    ct = orcs[0].encrypt(orcs[0].encode(rng.uniform(-1, 1, N // 2), 2.0 ** 40, ell), seed=4)
    sets = [[rng.uniform(-1, 1, N // 2) for _ in STEPS], [np.full(N // 2, 0.5) if i % 2 else None for i in range(len(STEPS))]]
    outs = []
    try:
        for t in (0, 1, 2):
            gks = [orcs[t].galois_key(o.galois_elt_from_step(N, s)) for s in STEPS]
            want, pts, flag = plain.lazy_rotsum(ct, list(STEPS), gks, sets, 2.0 ** 30)
            assert flag == 0
            w = [[pts.get((oi, i)) for i in range(len(STEPS))] for oi in range(len(sets))]
            be.select(bank, t)
            got = be.lazy_rotsum_with(ct, list(STEPS), gks, w)
            be.lib.emu_set_key_bank(None, C.c_size_t(0))
            pc.eq(got, want)
            outs.append(got)
    finally:
        be.lib.emu_set_key_bank(None, C.c_size_t(0))
    assert not np.array_equal(outs[0], outs[1]) and not np.array_equal(outs[1], outs[2])


# ---------------------------------------------------------------------------------------------------------------------------
# B200Server on the GPU: every instance against the oracle run with its own tenant's keys

ASSIGN = [0, 1, 2, 1, 0, 2]
PERMUTED = [2, 0, 1, 0, 2, 1]


class Fixture:
    """a golden program, 3 tenants with oracle keys of seeds 1..3 on one server, 6 instances with inputs of their own"""

    def __init__(self, name, seeds=(1, 2, 3), capacity=4):
        from eva_b200 import b200, program_io as gl
        from oracle_exec import OracleProgram
        self.d = d = gl.load_json(name)
        self.prog, self.params, _, self.terms = gl.build_program(d)
        N = d["poly_modulus_degree"]
        self.server = b200.B200Server(self.params, capacity=capacity)
        elts = self.server.bank_info()["galois_elements"]
        self.orcs, self.ops, self.keys = [], [], []
        for seed in seeds:
            orc = o.Oracle(N, d["prime_bits"]).keygen(seed)
            op = OracleProgram(d, orc)
            op.prepare_keys()
            op.gks.update({e: orc.galois_key(e) for e in elts if e not in op.gks})
            self.orcs.append(orc); self.ops.append(op)
            self.keys.append((op.rk, {int(e): op.gks[e] for e in elts}))
            assert self.server.add_raw_keys(*self.keys[-1]) == len(self.orcs) - 1
        self.vals, self.ins = [], []
        for i in range(len(ASSIGN)):
            v, io = self.valuation(self.orcs[ASSIGN[i] % len(self.orcs)], seed=40 + i)
            self.vals.append(v); self.ins.append(io)
        self._want = {}

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

    def check(self, outs, assign, what, instances=None):
        for i, out, t in zip(instances or range(len(outs)), outs, assign):
            V = self.want(i, t)
            for oname, oid in self.d["outputs"].items():
                kind, arr, scale = out.get(oname)
                if kind == "cipher":
                    assert np.array_equal(arr, V[oid][1]) and scale == V[oid][2], (what, i, t, oname)

    def drop_plans(self):
        for batch in (1, 2, 3):
            for r in range(len(ASSIGN)):
                self.server.drop_plan(self.prog, batch, r)

    def run(self, assign, **opts):
        if opts:
            self.server.set_options(**opts)
        return self.server.execute_batch(self.prog, list(zip(assign, self.vals)))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["sobel", "harris", "polynomial", "feat_mixed"])
def test_server_batches_bit_exact(name):
    """one execute_batch over 3 tenants, interleaved: every output the oracle's with the instance's own keys, for fuse 1, 2, 3 with
    and without the graph; every intermediate of a fused chunk; then a permuted assignment on the same plans, with no plan built
    and no launch issued (the captured graph reads the tenant table, it does not bake it in)"""
    f = Fixture(name)
    for graph in (True, False):
        f.drop_plans()   # use_graph and fuse_sums are fixed when a plan is built (not part of its staleness test)
        for fuse in (1, 2, 3):
            f.check(f.run(ASSIGN, fuse=fuse, use_graph=graph), ASSIGN, (graph, fuse))
            launches = f.server.launch_count()
            f.check(f.run(ASSIGN), ASSIGN, (graph, fuse, "repeated"))
            # a graph launch issues no kernel launch of its own; a replay without the graph issues every step again
            assert (f.server.launch_count() > launches) == (not graph), (graph, fuse)
    f.drop_plans()
    f.check(f.run(ASSIGN, fuse=3, use_graph=True, fuse_sums=False), ASSIGN, "materialised")
    for t in f.d["terms"]:
        for b in range(3):
            want = f.want(b, ASSIGN[b])[t["id"]]
            if want[0] == "raw":
                continue
            got = f.server.debug_value(f.prog, f.terms[t["id"]].index, 3, b)
            w = want[1] if want[0] == "cipher" else want[1][None]
            assert got is not None and np.array_equal(got[0], w), (name, b, t)
    built, launches = f.server.plans_built(), f.server.launch_count()
    f.check(f.run(PERMUTED), PERMUTED, "permuted")
    f.check(f.run(ASSIGN), ASSIGN, "again")
    assert f.server.plans_built() == built and f.server.launch_count() == launches


def _own_context(f, t, **opts):
    from eva_b200 import b200
    rk, gks = f.keys[t]
    pub = b200.context_from_raw_keys(f.d["poly_modulus_degree"], f.orcs[t].primes, rk, gks)
    pub.set_options(**opts)
    return pub


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_server_option_paths_match_each_tenants_context(name):
    """rotation_sums off, rotation chunks of 1 and 16, no shared mod-up, no hoisted rotations (evab_rotate_modup_prepared /
    evab_rotate_prepared / evab_rotate), a packed arena and approx_hoist: every instance equals its tenant's own B200Public
    under the same options, bit for bit (and the oracle where the options are exact)"""
    f = Fixture(name)
    unpacked = f.server.plan_stats(f.prog, 3, 0)["arena_bytes_unpacked"]
    pubs = [_own_context(f, t) for t in range(3)]
    for opts in (dict(rotation_sums=False), dict(rotation_chunk=1, rotation_sums=False), dict(rotation_chunk=16, rotation_sums=False),
                 dict(hoist_mod_up=False), dict(hoist_rotations=False), dict(arena_limit=unpacked - 1), dict(approx_hoist=True)):
        opts = dict(dict(fuse=3, rotation_sums=True, rotation_chunk=16, hoist_mod_up=True, hoist_rotations=True, arena_limit=0,
                         approx_hoist=False), **opts)
        outs = f.run(ASSIGN, **opts)
        for t in range(3):
            mine = [i for i, a in enumerate(ASSIGN) if a == t]
            pubs[t].set_options(**opts)
            ref = pubs[t].execute_batch(f.prog, [f.vals[i] for i in mine])
            for i, r in zip(mine, ref):
                for oname in f.d["outputs"]:
                    assert np.array_equal(outs[i].get(oname)[1], r.get(oname)[1]), (opts, i, oname)
        if not opts["approx_hoist"]:
            f.check(outs, ASSIGN, opts)
        assert f.server.plan_stats(f.prog, 3, 0)["packed"] == (opts["arena_limit"] > 0)


@pytest.mark.gpu
def test_server_zero_digit_falls_back():
    """one instance of tenant 1 has a zero digit coefficient (the shared mod-up does not hold for it) in a mixed batch: the
    batch is redone on the exact path and every instance returns the oracle's bits"""
    f = Fixture("sobel")
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
    for _ in range(2):
        f.check(f.run(ASSIGN, fuse=3), ASSIGN, "zero digit")


@pytest.mark.gpu
def test_server_garbage_keys_stay_with_their_tenant():
    """a tenant registered with uniformly random "keys", in the same fused batches as the others: every other instance is
    bit-identical to the oracle"""
    f = Fixture("sobel")
    rng = np.random.default_rng(99)
    k, N = f.orcs[0].k, f.d["poly_modulus_degree"]
    shape = (k - 1, 2, k, N)
    bad = f.server.add_raw_keys(rng.integers(0, 2 ** 60, shape, dtype=np.uint64),
                                {int(e): rng.integers(0, 2 ** 60, shape, dtype=np.uint64) for e in f.server.bank_info()["galois_elements"]})
    assert bad == 3
    assign = [0, bad, 1, bad, 2, bad]
    for fuse in (3, 2):
        outs = f.run(assign, fuse=fuse)
        mine = [i for i, t in enumerate(assign) if t != bad]
        f.check([outs[i] for i in mine], [assign[i] for i in mine], "isolation", mine)


@pytest.mark.gpu
def test_two_clients_user_flow():
    """two clients generate keys with different seeds and encrypt; the server registers their public contexts and runs one batch;
    each client decrypts its own outputs (MSE < 0.01 against evaluate); client A's output does not decrypt under client B's key"""
    from eva_b200 import EvaProgram, Input, Output, b200, evaluate
    from eva_b200.ckks import CKKSCompiler
    from eva_b200.metric import valuation_mse
    prog = EvaProgram("tenants", vec_size=256)
    with prog:
        x = Input("x")
        Output("y", x * (x << 1) + (x >> 3) * 0.5 - 1.0)
    prog.set_output_ranges(20)
    prog.set_input_scales(30)
    compiled, params, sig = CKKSCompiler().compile(prog)
    server = b200.B200Server(params, capacity=2)
    clients, requests, refs = [], [], []
    for c, seed in enumerate((11, 12)):
        pub, sec = b200.generate_keys(params, seed=seed)
        t = server.add_keys(pub)
        assert t == c
        for r in range(2):
            inputs = {"x": list(np.random.default_rng(100 * c + r).uniform(-1, 1, 256))}
            requests.append((t, pub.encrypt(inputs, sig)))
            refs.append((c, evaluate(compiled, inputs)))
        clients.append(sec)
    outs = server.execute_batch(compiled, requests)
    for out, (c, ref) in zip(outs, refs):
        assert valuation_mse(clients[c].decrypt(out, sig), ref) < 0.01
        assert valuation_mse(clients[1 - c].decrypt(out, sig), ref) > 0.01
    with pytest.raises(Exception):
        server.add_keys(b200.generate_keys(params, seed=13)[0])    # capacity 2: full


@pytest.mark.gpu
def test_server_errors():
    from eva_b200 import b200
    from eva_b200.ckks import CKKSParameters as b200_params
    f = Fixture("polynomial", seeds=(1, 2), capacity=2)
    rk, gks = f.keys[0]
    with pytest.raises(Exception, match="full"):
        f.server.add_raw_keys(rk, gks)
    for bad in (5, -1):
        with pytest.raises(Exception):
            f.server.execute(f.prog, bad, f.vals[0])
    with pytest.raises(Exception, match="does not match"):
        f.server.add_raw_keys(rk[:, :, :-1], gks)
    # a server that rotates needs every Galois element of its rotation set
    s = Fixture("feat_rot_m1", seeds=(1,))
    rk1, gks1 = s.keys[0]
    missing = next(iter(gks1))
    with pytest.raises(Exception, match=str(missing)):
        s.server.add_raw_keys(rk1, {e: k for e, k in gks1.items() if e != missing})
    with pytest.raises(Exception, match="does not match"):
        s.server.add_raw_keys(rk1, {e: k[:, :, :, :-1] for e, k in gks1.items()})
    # a context with other primes
    other, _ = b200.generate_keys(b200_params([40] + list(s.params.prime_bits)[1:], s.params.rotations, s.d["poly_modulus_degree"]), seed=3)
    with pytest.raises(Exception, match="N / primes"):
        s.server.add_keys(other)
    # removal: unknown ids, then a tenant used by a batch that is not collected
    f.server.remove_keys(1)
    with pytest.raises(Exception):
        f.server.remove_keys(1)
    with pytest.raises(Exception):
        f.server.execute(f.prog, 1, f.vals[1])
    h = f.server.execute_batch_async(f.prog, [(0, f.vals[0])], 0)
    with pytest.raises(Exception, match="not been collected"):
        f.server.remove_keys(0)
    f.check(f.server.execute_batch_result(h), [0], "async")
    f.server.remove_keys(0)
    assert f.server.bank_info()["tenants"] == 0
