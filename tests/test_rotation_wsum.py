"""Bit-exact weighted rotation sums (evab_rotate_wsum): the kernels on the CPU emulator and the GPU against the oracle, and the
executor's rotation_sums plans (the default) against plans without them."""
import ctypes as C

import numpy as np
import pytest

import parity_cases as pc
from backends import EmuBackend, GpuBackend, _elt, _p
from oracle import oracle as o


def _ptrs(xs):
    return (C.c_void_p * max(1, len(xs)))(*xs)


class WsumEmuBackend(EmuBackend):
    """EmuBackend plus evab_rotate_wsum replayed on the CPU (tests/emu/emu_wsum.cpp: emu.cpp + the new kernel body and the forward
    NTT with PRO_PLAIN + EPI_DIVROUND), in a library and context of its own"""
    SRC, LIB = "emu_wsum.cpp", "libevab_emu_wsum"

    def __init__(self, N, primes, bound_check=False):
        super().__init__(N, primes, bound_check=bound_check)
        for fn in ("emu_rotate_modup_work_bytes", "emu_rotate_wsum_work_bytes"):
            getattr(self.lib, fn).restype = C.c_size_t

    def rotate_wsum(self, a, steps_list, gks, wts, taps, twts):
        """out_o = sum_i wts[o][i] (.) rotate(a, steps[i]) + sum_t twts[o][t] (.) taps[t] (scalar plaintexts [ell][N], None: weight 0).
        Returns (outs [nout][2][ell][N], zero flag)"""
        lib, h, N = self.lib, self.h, self.N
        ell = a.shape[1]
        that = np.empty((ell, N), dtype=np.uint64)
        ext = np.zeros((ell + 1, ell, N), dtype=np.uint64)
        zflag = np.zeros(1, dtype=np.uint64)
        self._chk(lib.emu_rotate_modup_prepare(h, ell, _p(that), _p(ext), _p(a), _p(zflag)))
        self._chk(lib.emu_rotate_modup_scale_c0(h, ell, _p(ext), _p(a)))
        n, nout = len(steps_list), len(wts)
        cadds = []
        for s_, gk in zip(steps_list, gks):
            cadd = np.empty((2, ell + 1, N), dtype=np.uint64)
            tmp = np.empty((ell + 1, N), dtype=np.uint64)
            self._chk(lib.emu_rotate_hoist_const(h, ell, C.c_uint64(_elt(N, s_)), _p(gk), _p(cadd), _p(tmp)))
            cadds.append(cadd)
        keep = [np.ascontiguousarray(x) for x in list(gks) + list(taps)]
        plains = [[None if w is None else np.ascontiguousarray(w) for w in ws] for ws in list(wts) + list(twts)]
        ptr = lambda x: None if x is None else x.ctypes.data
        work = np.zeros(lib.emu_rotate_wsum_work_bytes(h, ell, n, nout) // 8, dtype=np.uint64)
        out = np.empty((nout, 2, ell, N), dtype=np.uint64)
        self._chk(lib.emu_rotate_wsum(h, ell, nout, _p(out), _p(a), _p(ext), n, (C.c_uint64 * n)(*[_elt(N, s_) for s_ in steps_list]),
                                      _ptrs([g.ctypes.data for g in keep[:n]]), _ptrs([c_.ctypes.data for c_ in cadds]),
                                      _ptrs([ptr(w) for ws in plains[:nout] for w in ws]), len(taps), _ptrs([t.ctypes.data for t in keep[n:]]),
                                      _ptrs([ptr(w) for ws in plains[nout:] for w in ws]), _p(work)))
        return out, int(zflag[0])


class WsumGpuBackend(GpuBackend):
    """GpuBackend plus evab_rotate_wsum through the C-ABI"""

    def rotate_wsum(self, a, steps_list, gks, wts, taps, twts):
        lib = self.lib
        ell = a.shape[1]
        da = self._up(a)
        that = self._alloc(ell * self.N * 8)
        ext = self._alloc(lib.evab_rotate_modup_ext_bytes(self.h, ell))
        zf = self._alloc(8)
        self._chk(lib.evab_memset_zero(self.h, zf, 8, None))
        self._chk(lib.evab_rotate_modup_prepare(self.h, ell, that, ext, da, zf, None))
        self._chk(lib.evab_rotate_modup_scale_c0(self.h, ell, ext, da, None))
        n, nout = len(steps_list), len(wts)
        elts, dks, dcs = [], [], []
        for s_, gk in zip(steps_list, gks):
            elt = _elt(self.N, s_)
            if elt not in self._prepared:
                self._chk(lib.evab_galois_prepare(self.h, C.c_uint64(elt)))
                self._prepared.add(elt)
            dk = self._up(gk)
            cadd = self._alloc(lib.evab_hoist_const_bytes(self.h, ell))
            tmp = self._alloc((ell + 1) * self.N * 8)
            self._chk(lib.evab_rotate_hoist_const(self.h, ell, C.c_uint64(elt), dk, cadd, tmp, None))
            elts.append(elt); dks.append(dk); dcs.append(cadd)
            self._free(tmp)
        dts = [self._up(t) for t in taps]
        dws = [[None if w is None else self._up(w) for w in ws] for ws in list(wts) + list(twts)]
        work = self._alloc(lib.evab_rotate_wsum_work_bytes(self.h, ell, n, nout))
        do = self._alloc(nout * 2 * ell * self.N * 8)
        self._chk(lib.evab_rotate_wsum(self.h, ell, nout, do, da, ext, n, (C.c_uint64 * n)(*elts), _ptrs(dks), _ptrs(dcs),
                                       _ptrs([w for ws in dws[:nout] for w in ws]), len(taps), _ptrs(dts),
                                       _ptrs([w for ws in dws[nout:] for w in ws]), work, None))
        out = self._down(do, (nout, 2, ell, self.N))
        flag = int(self._down(zf, (1,))[0])
        self._free(da, that, ext, zf, work, do, *dks, *dcs, *dts, *[w for ws in dws for w in ws if w is not None])
        return out, flag


WSUM_STEPS = (1, -1, 2, 7, 64, -3, 5, 100, 31, -64, 9, 13, 200, -7, 17, 33)
WSUM_VALUES = (1.0, -2.0, 0.0, 0.5, -0.25, 3.0, 2.213787482387662, -1.0984324107372518, -1.0, 2.0)


def case_rotation_wsum(be, orc, ell, n, nout, seed=0):
    """evab_rotate_wsum: out_o = sum_i w_oi (.) rotate(x, s_i) + sum_t v_ot (.) tap_t with scalar plaintext weights (some 0.0, some
    negative, some absent) == the oracle's rotate -> multiply_plain -> add, word for word.  The taps are x itself (a rotation by 0
    folded into the sum) and a second ciphertext."""
    x, y = pc.rand_ct(orc, 2, ell, 800 + seed), pc.rand_ct(orc, 2, ell, 900 + seed)
    steps = WSUM_STEPS[:n]
    gks = [orc.galois_key(o.galois_elt_from_step(orc.N, s)) for s in steps]
    enc = {}

    def pt(v):
        if v not in enc:
            enc[v] = orc.encode(np.array([v]), 2.0 ** 30, ell)
        return enc[v]
    pick = lambda o_, i: (o_ * 7 + i * 3 + seed) % (len(WSUM_VALUES) + 1)
    wts = [[None if pick(o_, i) == len(WSUM_VALUES) else pt(WSUM_VALUES[pick(o_, i)]) for i in range(n)] for o_ in range(nout)]
    taps = [x, y]
    twts = [[pt(-1.0 - o_), None if o_ % 2 else pt(0.5 * o_ - 0.75)] for o_ in range(nout)]
    outs, flag = be.rotate_wsum(x, list(steps), gks, wts, taps, twts)
    assert flag == 0
    rots = [orc.rotate(x, s, gk) for s, gk in zip(steps, gks)]
    for o_ in range(nout):
        want = None
        for c, w in list(zip(rots, wts[o_])) + list(zip(taps, twts[o_])):
            if w is not None:
                term = orc.mul_plain(c, w)
                want = term if want is None else orc.add(want, term)
        pc.eq(outs[o_], want)


# (ell, rotations, sums): ell in {1, 2, k-1}, n in {1, 8, 16}, nout in {1, 2, 4}
SHAPES = [(1, 1, 1), (2, 8, 2), (3, 16, 4), (3, 8, 4), (1, 16, 2)]


@pytest.mark.parametrize("ell,n,nout", SHAPES)
def test_rotation_wsum_emulated(ell, n, nout):
    orc = pc.get_oracle(1024, [60, 60, 60, 60])
    case_rotation_wsum(WsumEmuBackend(1024, orc.primes), orc, ell, n, nout)


def test_rotation_wsum_emulated_mixed_primes():
    """a key-switch prime much larger than the residue primes: P mod q_r and tmp mod q_r are real reductions"""
    orc = pc.get_oracle(1024, [60, 40, 40, 60])
    case_rotation_wsum(WsumEmuBackend(1024, orc.primes), orc, 2, 8, 2, seed=3)


@pytest.mark.gpu
@pytest.mark.parametrize("ell,n,nout", SHAPES)
def test_rotation_wsum_gpu_small(ell, n, nout):
    orc = pc.get_oracle(1024, [60, 60, 60, 60])
    case_rotation_wsum(WsumGpuBackend(1024, orc.primes), orc, ell, n, nout)


@pytest.mark.gpu
@pytest.mark.parametrize("ell,n,nout", [(4, 8, 2), (1, 16, 4), (2, 1, 1), (4, 16, 4)])
def test_rotation_wsum_gpu_sobel_shape(ell, n, nout):
    orc = pc.get_oracle(16384, [60] * 5)
    case_rotation_wsum(WsumGpuBackend(16384, orc.primes), orc, ell, n, nout, seed=1)


# ---- executor: rotation_sums plans (the default) against plans without them and against the oracle

def _context(d, seed=1):
    from eva_b200 import b200
    from oracle import oracle as o
    from oracle_exec import OracleProgram
    N = d["poly_modulus_degree"]
    orc = o.Oracle(N, d["prime_bits"]).keygen(seed)
    op = OracleProgram(d, orc)
    op.prepare_keys()
    pub = b200.context_from_raw_keys(N, orc.primes, op.rk, {int(e): k for e, k in op.gks.items()})
    return orc, op, pub


def _valuation(d, orc, seed=5):
    from eva_b200 import b200
    rng = np.random.default_rng(seed)
    val, inputs_o = b200.B200Valuation(), {}
    for name, info in d["signature"].items():
        x = rng.uniform(0.0, 0.2, d["vec_size"])
        ell, scale = orc.k - 1 - info["level"], 2.0 ** info["scale"]
        if info["type"] == "Cipher":
            ct = orc.encrypt(orc.encode(x, scale, ell), seed=seed)
            val.set_cipher(name, ct, scale); inputs_o[name] = ("cipher", ct, scale)
        elif info["type"] == "Raw":
            val.set_raw(name, list(x)); inputs_o[name] = ("raw", x)
        else:
            pt = orc.encode(x, scale, ell)
            val.set_plain(name, pt, scale); inputs_o[name] = ("plain", pt, scale)
    return val, inputs_o


def _run(d, **opts):
    """outputs of rotation_sums on and off (execute twice: the second replays the captured graph), both checked against the oracle
    word for word; returns the plan statistics of each setting"""
    from eva_b200 import program_io as gl
    prog, _, _, terms = gl.build_program(d)
    orc, op, pub = _context(d)
    val, inputs_o = _valuation(d, orc)
    V = op.run(inputs_o)
    stats = {}
    for on in (True, False):
        pub.set_options(rotation_sums=on, **opts)
        for _ in range(2):
            out = pub.execute(prog, val)
            for oname, oid in d["outputs"].items():
                kind, arr, scale = out.get(oname)
                if kind == "cipher":
                    assert np.array_equal(arr, V[oid][1]) and scale == V[oid][2], (oname, on)
        stats[on] = pub.plan_stats(prog)
        for t in d["terms"]:   # every value the plan materialises is the oracle's
            got = pub.debug_value(prog, terms[t["id"]].index)
            if got is not None and V[t["id"]][0] == "cipher":
                assert np.array_equal(got[0], V[t["id"]][1]), (t, on)
    return stats


FEATURES = ["feat_bin_mul_11", "feat_bin_sub_01", "feat_unary", "feat_rot_m1", "feat_rot_0", "feat_mixed", "feat_transparent",
            "feat_hsum", "feat_deep", "polynomial", "wide64"]


@pytest.mark.gpu
@pytest.mark.parametrize("cache", [True, False])
@pytest.mark.parametrize("name", ["sobel", "harris"] + FEATURES)
def test_rotation_sums_executor_parity(name, cache):
    from eva_b200 import program_io as gl
    st = _run(gl.load_json(name), cache_constants=cache)
    assert st[False]["rotation_sum_calls"] == 0
    if name in ("sobel", "harris"):
        assert st[True]["rotation_sum_calls"] > 0 and st[True]["steps"] < st[False]["steps"]


@pytest.mark.gpu
def test_sobel_plan_is_one_call():
    """Sobel's two filters over the 8 rotations of the image: one call of 2 sums over 7 rotations (rotation 65 has weight 0.0 in both
    and is never computed), the rotation-0 taps folded in through the image itself, no materialised rotation left"""
    from eva_b200 import program_io as gl
    d = gl.load_json("sobel")
    prog, _, _, terms = gl.build_program(d)
    _, _, pub = _context(d)
    st = pub.plan_stats(prog)
    assert (st["rotation_sum_calls"], st["rotation_sums"], st["rotation_sum_rotations"], st["rotation_sum_taps"]) == (1, 2, 7, 1), st
    assert st["chunked_rotations"] == 0 and st["rotation_chunks"] == 0 and st["lazy_calls"] == 0
    rot = {t["rotation"]: t["id"] for t in d["terms"] if t["op"] == "RotateLeftConst"}
    assert st["elided_rotations"] == len(rot) == 9
    assert pub.debug_value(prog, terms[rot[65]].index) is None


@pytest.mark.gpu
def test_vector_weights_keep_the_chunk_path():
    """weights that are not replicated scalars (here: every constant of Sobel made a vector) leave the rotations on the
    materialised path; results still the oracle's"""
    import copy
    from eva_b200 import program_io as gl
    d = copy.deepcopy(gl.load_json("sobel"))
    for t in d["terms"]:
        if t["op"] == "Constant" and t["level"] == 3:
            t["const"] = [t["const"][0], t["const"][0] + 0.125] * 4
    st = _run(d)
    assert st[True]["rotation_sum_calls"] == 0 and st[True]["chunked_rotations"] == 8 and st[True]["steps"] == st[False]["steps"]


@pytest.mark.gpu
def test_rotation_sums_packed_and_batched():
    """the call's outputs in a packed arena and in fused batches: the bits of the unpacked single-instance plan"""
    from eva_b200 import b200, program_io as gl
    for name in ("sobel", "harris"):
        d = gl.load_json(name)
        prog, _, _, _ = gl.build_program(d)
        orc, op, pub = _context(d)
        vals = [_valuation(d, orc, seed=7 + i) for i in range(3)]
        want = [op.run(io_) for _, io_ in vals]
        unpacked = pub.plan_stats(prog, 3, 0)["arena_bytes_unpacked"]
        for opts in (dict(fuse=3), dict(fuse=3, arena_limit=unpacked - 1), dict(fuse=1, cache_constants=False)):
            pub.set_options(**opts)
            outs = pub.execute_batch(prog, [v for v, _ in vals])
            for out, V in zip(outs, want):
                for oname, oid in d["outputs"].items():
                    assert np.array_equal(out.get(oname)[1], V[oid][1]), (name, opts)
        assert pub.plan_stats(prog, 3, 0)["rotation_sum_calls"] > 0
