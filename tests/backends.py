"""Numpy-in / numpy-out drivers for the two implementations of the C-ABI ops:

* ``EmuBackend``  -- CPU replay of the CUDA kernel bodies (tests/emu/emu.cpp)
* ``GpuBackend``  -- the real product library ``eva_b200/lib/libevab200.so``
                     through include/evab200.h (device buffers + streams)

Both expose the same methods as ``oracle.oracle.Oracle`` so the parity cases in
tests/parity_cases.py run unchanged against either.
"""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
u64p = C.POINTER(C.c_uint64)


def _p(a):
    assert a.dtype == np.uint64 and a.flags.c_contiguous
    return a.ctypes.data_as(u64p)


def _elt(N, steps):
    m = 2 * N
    if steps == 0:
        return m - 1
    s = steps if steps > 0 else N // 2 - (-steps)
    return pow(3, s, m)


class EmuBackend:
    name = "emu"
    SRC, LIB = "emu.cpp", "libevab_emu"     # source under tests/emu and the library it builds

    def __init__(self, N, primes, cluster=1, bound_check=False):
        """bound_check: a separately built library with -DEVAB_BOUND_CHECK, in which every compile-time bound of the fold
        arithmetic is checked against the value it describes; a violated bound prints `bound violated at ...` and aborts the
        process, so run it in a subprocess"""
        so = os.path.join(ROOT, "tests", "emu", self.LIB + ("_bc.so" if bound_check else ".so"))
        src = os.path.join(ROOT, "tests", "emu", self.SRC)
        deps = [src, os.path.join(ROOT, "tests", "emu", "emu.cpp")] + [os.path.join(ROOT, "eva_b200", "csrc", f) for f in os.listdir(os.path.join(ROOT, "eva_b200", "csrc"))]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            defs = ["-DEVAB_BOUND_CHECK"] if bound_check else []
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off"] + defs + ["-x", "c++", src, "-o", so])
        self.lib = C.CDLL(so)
        assert self.lib.emu_bound_checked() == int(bound_check)
        self.lib.emu_ctx_create.restype = C.c_void_p
        self.lib.emu_last_error.restype = C.c_char_p
        for n in ("emu_rescale_work_bytes", "emu_keyswitch_work_bytes", "emu_encode_work_bytes"):
            getattr(self.lib, n).restype = C.c_size_t
        pa = np.array(primes, dtype=np.uint64)
        self.h = C.c_void_p(self.lib.emu_ctx_create(C.c_uint64(N), _p(pa), len(primes)))
        if not self.h:
            raise RuntimeError(self.lib.emu_last_error().decode())
        self.N, self.k = N, len(primes)
        self.cluster = cluster

    def _chk(self, rc):
        if rc:
            raise RuntimeError(self.lib.emu_last_error().decode())

    def __getattribute__(self, name):
        # the emulator's cluster setting is process-global: select this backend's value before every op
        if name in ("ntt", "rescale", "relinearize", "rotate", "rotate_many", "encode"):
            object.__getattribute__(self, "lib").emu_set_cluster(object.__getattribute__(self, "cluster"))
        return object.__getattribute__(self, name)

    def ntt(self, data, prime_idx, inverse=False):
        d = np.ascontiguousarray(data, dtype=np.uint64).copy()
        flat = d.reshape(-1, self.N)
        arr = (C.c_int * len(prime_idx))(*prime_idx)
        fn = self.lib.emu_ntt_inv if inverse else self.lib.emu_ntt_fwd
        self._chk(fn(self.h, _p(d), C.c_size_t(flat.shape[0]), arr, len(prime_idx)))
        return d

    def _bin(self, fn, a, b):
        out = np.empty((max(a.shape[0], b.shape[0]), a.shape[1], self.N), dtype=np.uint64)
        self._chk(getattr(self.lib, fn)(self.h, a.shape[1], _p(out), _p(a), a.shape[0], _p(b), b.shape[0]))
        return out

    def add(self, a, b): return self._bin("emu_add", a, b)
    def sub(self, a, b): return self._bin("emu_sub", a, b)

    def _plain(self, fn, a, pt):
        out = np.empty_like(a)
        self._chk(getattr(self.lib, fn)(self.h, a.shape[1], _p(out), _p(a), a.shape[0], _p(pt)))
        return out

    def add_plain(self, a, pt): return self._plain("emu_add_plain", a, pt)
    def sub_plain(self, a, pt): return self._plain("emu_sub_plain", a, pt)
    def mul_plain(self, a, pt): return self._plain("emu_mul_plain", a, pt)

    def sum_terms(self, cts, pts):
        """out = sum_t (pts[t] is None ? cts[t] : cts[t] * pts[t])"""
        n = len(cts)
        ell = cts[0].shape[1]
        out = np.empty((max(c.shape[0] for c in cts), ell, self.N), dtype=np.uint64)
        cp = (C.c_void_p * n)(*[c.ctypes.data for c in cts])
        pp = (C.c_void_p * n)(*[(p.ctypes.data if p is not None else None) for p in pts])
        sz = (C.c_int * n)(*[c.shape[0] for c in cts])
        self._chk(self.lib.emu_sum_terms(self.h, ell, _p(out), n, cp, sz, pp))
        return out

    def sum_products(self, cts, seconds, kinds):
        """terms of kind 0 (ct), 1 (ct * plaintext) or 2 (ct (x) ct)"""
        n = len(cts)
        ell = cts[0].shape[1]
        sout = max(3 if k == 2 else c.shape[0] for c, k in zip(cts, kinds))
        out = np.empty((sout, ell, self.N), dtype=np.uint64)
        cp = (C.c_void_p * n)(*[c.ctypes.data for c in cts])
        pp = (C.c_void_p * n)(*[(p.ctypes.data if p is not None else None) for p in seconds])
        sz = (C.c_int * n)(*[c.shape[0] for c in cts])
        kd = (C.c_int * n)(*kinds)
        self._chk(self.lib.emu_sum_products(self.h, ell, _p(out), n, cp, sz, pp, kd))
        return out

    def negate(self, a):
        out = np.empty_like(a)
        self._chk(self.lib.emu_negate(self.h, a.shape[1], _p(out), _p(a), a.shape[0]))
        return out

    def mul(self, a, b):
        out = np.empty((3, a.shape[1], self.N), dtype=np.uint64)
        self._chk(self.lib.emu_mul(self.h, a.shape[1], _p(out), _p(a), _p(b)))
        return out

    def square(self, a):
        out = np.empty((3, a.shape[1], self.N), dtype=np.uint64)
        self._chk(self.lib.emu_square(self.h, a.shape[1], _p(out), _p(a)))
        return out

    def rescale(self, a):
        out = np.empty((a.shape[0], a.shape[1] - 1, self.N), dtype=np.uint64)
        work = np.zeros(self.lib.emu_rescale_work_bytes(self.h, a.shape[0]) // 8, dtype=np.uint64)
        self._chk(self.lib.emu_rescale(self.h, a.shape[1], _p(out), _p(a), a.shape[0], _p(work)))
        return out

    def mod_switch(self, a):
        return np.ascontiguousarray(a[:, :-1])

    def relinearize(self, a, rk):
        out = np.empty((2, a.shape[1], self.N), dtype=np.uint64)
        work = np.zeros(self.lib.emu_keyswitch_work_bytes(self.h, a.shape[1]) // 8, dtype=np.uint64)
        self._chk(self.lib.emu_relinearize(self.h, a.shape[1], _p(out), _p(a), _p(rk), _p(work)))
        return out

    def rotate(self, a, steps, gk):
        out = np.empty((2, a.shape[1], self.N), dtype=np.uint64)
        work = np.zeros(self.lib.emu_keyswitch_work_bytes(self.h, a.shape[1]) // 8, dtype=np.uint64)
        self._chk(self.lib.emu_rotate(self.h, a.shape[1], _p(out), _p(a), C.c_uint64(_elt(self.N, steps)), _p(gk), _p(work)))
        return out

    def encode(self, values, scale, ell):
        """Batched-encoder kernel bodies on the CPU: list of vectors (or one vector) -> [count][ell][N]."""
        single = np.ndim(values[0]) == 0
        vecs = [np.ascontiguousarray(values, dtype=np.float64)] if single else [np.ascontiguousarray(v, dtype=np.float64) for v in values]
        n = len(vecs)
        ptrs = (C.c_void_p * n)(*[v.ctypes.data for v in vecs])
        sizes = (C.c_uint32 * n)(*[len(v) for v in vecs])
        scales = (C.c_double * n)(*([float(scale)] * n))
        out = np.empty((n, ell, self.N), dtype=np.uint64)
        work = np.zeros(self.lib.emu_encode_work_bytes(self.h, n) // 8, dtype=np.uint64)
        self._chk(self.lib.emu_encode(self.h, n, ptrs, sizes, scales, ell, _p(out), _p(work)))
        return out[0] if single else out

    def encode_uniform(self, values, scale, ell):
        """scalar constants: [count] values -> [count][ell][N] (evab_encode_uniform)"""
        n = len(values)
        vals = (C.c_double * n)(*[float(v) for v in values])
        scales = (C.c_double * n)(*([float(scale)] * n))
        out = np.empty((n, ell, self.N), dtype=np.uint64)
        self._chk(self.lib.emu_encode_uniform(self.h, n, vals, scales, ell, _p(out)))
        return out

    def rotate_many(self, a, steps_list, gks):
        """rotations of one ciphertext sharing the inverse NTT of c1 (evab_rotate_prepare / _prepared)"""
        ell = a.shape[1]
        hoist = np.empty((ell, self.N), dtype=np.uint64)
        self._chk(self.lib.emu_rotate_prepare(self.h, ell, _p(hoist), _p(a)))
        outs = []
        for s_, gk in zip(steps_list, gks):
            out = np.empty((2, ell, self.N), dtype=np.uint64)
            work = np.zeros(self.lib.emu_keyswitch_work_bytes(self.h, ell) // 8, dtype=np.uint64)
            self._chk(self.lib.emu_rotate_prepared(self.h, ell, _p(out), _p(a), _p(hoist), C.c_uint64(_elt(self.N, s_)), _p(gk), _p(work)))
            outs.append(out)
        return outs

    def decode(self, pt, scale, primes):
        out = np.empty(self.N // 2, dtype=np.float64)
        pa = np.array(primes, dtype=np.uint64)
        self._chk(self.lib.emu_decode(self.h, pt.shape[0], _p(pa), _p(np.ascontiguousarray(pt)), C.c_double(scale), out.ctypes.data_as(C.c_void_p)))
        return out

    def rotate_many_modup(self, a, steps_list, gks):
        """rotations of one ciphertext sharing inverse NTT AND mod-up (evab_rotate_modup_*): (outputs, zero flag)"""
        ell = a.shape[1]
        that = np.empty((ell, self.N), dtype=np.uint64)
        ext = np.zeros((ell + 1, ell, self.N), dtype=np.uint64)
        zflag = np.zeros(1, dtype=np.uint64)
        self._chk(self.lib.emu_rotate_modup_prepare(self.h, ell, _p(that), _p(ext), _p(a), _p(zflag)))
        self.lib.emu_rotate_modup_work_bytes.restype = C.c_size_t
        outs = []
        for s_, gk in zip(steps_list, gks):
            elt = C.c_uint64(_elt(self.N, s_))
            cadd = np.empty((2, ell + 1, self.N), dtype=np.uint64)
            tmp = np.empty((ell + 1, self.N), dtype=np.uint64)
            self._chk(self.lib.emu_rotate_hoist_const(self.h, ell, elt, _p(gk), _p(cadd), _p(tmp)))
            out = np.empty((2, ell, self.N), dtype=np.uint64)
            work = np.zeros(self.lib.emu_rotate_modup_work_bytes(self.h, ell) // 8, dtype=np.uint64)
            self._chk(self.lib.emu_rotate_modup_prepared(self.h, ell, _p(out), _p(a), _p(ext), elt, _p(gk), _p(cadd), _p(work)))
            outs.append(out)
        # the same rotations in one call (evab_rotate_modup_many)
        n = len(steps_list)
        cadds = []
        for s_, gk in zip(steps_list, gks):
            cadd = np.empty((2, ell + 1, self.N), dtype=np.uint64)
            tmp = np.empty((ell + 1, self.N), dtype=np.uint64)
            self._chk(self.lib.emu_rotate_hoist_const(self.h, ell, C.c_uint64(_elt(self.N, s_)), _p(gk), _p(cadd), _p(tmp)))
            cadds.append(cadd)
        gkc = [np.ascontiguousarray(g) for g in gks]
        self._chk(self.lib.emu_rotate_modup_scale_c0(self.h, ell, _p(ext), _p(a)))
        self.lib.emu_rotate_modup_many_work_bytes.restype = C.c_size_t
        mw = np.zeros(self.lib.emu_rotate_modup_many_work_bytes(self.h, ell, n) // 8, dtype=np.uint64)
        many = np.empty((n, 2, ell, self.N), dtype=np.uint64)
        self._chk(self.lib.emu_rotate_modup_many(self.h, ell, n, _p(many), _p(a), _p(ext), (C.c_uint64 * n)(*[_elt(self.N, s_) for s_ in steps_list]),
                                                 (C.c_void_p * n)(*[g.ctypes.data for g in gkc]), (C.c_void_p * n)(*[c_.ctypes.data for c_ in cadds]), _p(mw)))
        self.many = [many[i] for i in range(n)]
        return outs, int(zflag[0])

    def lazy_rotsum(self, a, steps_list, gks, weight_sets, scale):
        """out_o = sum_i encode(weight_sets[o][i]) (.) rotate(a, steps[i]) (None: rotation i not in sum o) with ONE mod-down per
        sum (evab_lazy_rotsum; approximate by design).  Returns (outs [nout][2][ell][N], plaintexts {(o, i): [ell+1][N]}, zero flag)"""
        ell = a.shape[1]
        that = np.empty((ell, self.N), dtype=np.uint64)
        ext = np.zeros((ell + 1, ell, self.N), dtype=np.uint64)
        zflag = np.zeros(1, dtype=np.uint64)
        self._chk(self.lib.emu_rotate_modup_prepare(self.h, ell, _p(that), _p(ext), _p(a), _p(zflag)))
        self._chk(self.lib.emu_rotate_modup_scale_c0(self.h, ell, _p(ext), _p(a)))
        n, nout = len(steps_list), len(weight_sets)
        where = [(o, i) for o in range(nout) for i in range(n) if weight_sets[o][i] is not None]
        vecs = [np.ascontiguousarray(weight_sets[o][i], dtype=np.float64) for o, i in where]
        m = len(vecs)
        ptrs = (C.c_void_p * m)(*[v.ctypes.data for v in vecs])
        sizes = (C.c_uint32 * m)(*[len(v) for v in vecs])
        scales = (C.c_double * m)(*([float(scale)] * m))
        pts = np.empty((m, ell + 1, self.N), dtype=np.uint64)
        work = np.zeros(self.lib.emu_encode_work_bytes(self.h, m) // 8, dtype=np.uint64)
        self._chk(self.lib.emu_encode_ext(self.h, m, ptrs, sizes, scales, ell, 1, _p(pts), _p(work)))
        cadds = []
        for s_, gk in zip(steps_list, gks):
            cadd = np.empty((2, ell + 1, self.N), dtype=np.uint64)
            tmp = np.empty((ell + 1, self.N), dtype=np.uint64)
            self._chk(self.lib.emu_rotate_hoist_const(self.h, ell, C.c_uint64(_elt(self.N, s_)), _p(gk), _p(cadd), _p(tmp)))
            cadds.append(cadd)
        elts = (C.c_uint64 * n)(*[_elt(self.N, s_) for s_ in steps_list])
        gks = [np.ascontiguousarray(g) for g in gks]
        keys = (C.c_void_p * n)(*[g.ctypes.data for g in gks])
        cads = (C.c_void_p * n)(*[c_.ctypes.data for c_ in cadds])
        wl = [None] * (nout * n)
        for idx, (o, i) in enumerate(where):
            wl[o * n + i] = pts[idx].ctypes.data
        wts = (C.c_void_p * (nout * n))(*wl)
        self.lib.emu_lazy_rotsum_work_bytes.restype = C.c_size_t
        lw = np.zeros(self.lib.emu_lazy_rotsum_work_bytes(self.h, ell, nout) // 8, dtype=np.uint64)
        out = np.empty((nout, 2, ell, self.N), dtype=np.uint64)
        self._chk(self.lib.emu_lazy_rotsum(self.h, ell, nout, _p(out), _p(a), _p(ext), n, elts, keys, cads, wts, _p(lw)))
        return out, {oi: pts[idx] for idx, oi in enumerate(where)}, int(zflag[0])

class GpuBackend:
    """Calls the product C-ABI (include/evab200.h).  Fails loudly if the CUDA
    extension is missing -- there is no fallback."""
    name = "gpu"

    def __init__(self, N, primes, device=0):
        from eva_b200 import cabi
        self.lib = cabi.load()
        pa = np.array(primes, dtype=np.uint64)
        h = C.c_void_p()
        self._chk(self.lib.evab_ctx_create(C.c_uint64(N), _p(pa), len(primes), device, C.byref(h)))
        self.h = h
        self.N, self.k = N, len(primes)
        self._prepared = set()

    def __del__(self):
        try:
            self.lib.evab_ctx_destroy(self.h)
        except Exception:
            pass

    def _chk(self, rc):
        if rc:
            raise RuntimeError(self.lib.evab_last_error().decode())

    def _up(self, a):
        a = np.ascontiguousarray(a, dtype=np.uint64)
        d = C.c_void_p()
        self._chk(self.lib.evab_malloc(self.h, C.c_size_t(a.nbytes), C.byref(d), None))
        self._chk(self.lib.evab_upload(self.h, d, a.ctypes.data_as(C.c_void_p), C.c_size_t(a.nbytes), None))
        return d

    def _alloc(self, nbytes):
        d = C.c_void_p()
        self._chk(self.lib.evab_malloc(self.h, C.c_size_t(nbytes), C.byref(d), None))
        return d

    def _down(self, d, shape):
        out = np.empty(shape, dtype=np.uint64)
        self._chk(self.lib.evab_download(self.h, out.ctypes.data_as(C.c_void_p), d, C.c_size_t(out.nbytes), None))
        self._chk(self.lib.evab_sync(self.h, None))
        return out

    def _free(self, *ds):
        for d in ds:
            self._chk(self.lib.evab_free(self.h, d, None))

    def ntt(self, data, prime_idx, inverse=False):
        shape = np.asarray(data).shape
        d = self._up(data)
        arr = (C.c_int * len(prime_idx))(*prime_idx)
        cnt = int(np.prod(shape)) // self.N
        fn = self.lib.evab_ntt_inv if inverse else self.lib.evab_ntt_fwd
        self._chk(fn(self.h, d, C.c_size_t(cnt), arr, len(prime_idx), None))
        out = self._down(d, shape)
        self._free(d)
        return out

    def _bin(self, fn, a, b):
        shape = (max(a.shape[0], b.shape[0]), a.shape[1], self.N)
        da, db, do = self._up(a), self._up(b), self._alloc(int(np.prod(shape)) * 8)
        self._chk(getattr(self.lib, fn)(self.h, a.shape[1], do, da, a.shape[0], db, b.shape[0], None))
        out = self._down(do, shape)
        self._free(da, db, do)
        return out

    def add(self, a, b): return self._bin("evab_add", a, b)
    def sub(self, a, b): return self._bin("evab_sub", a, b)

    def _plain(self, fn, a, pt):
        da, dp, do = self._up(a), self._up(pt), self._alloc(a.nbytes)
        self._chk(getattr(self.lib, fn)(self.h, a.shape[1], do, da, a.shape[0], dp, None))
        out = self._down(do, a.shape)
        self._free(da, dp, do)
        return out

    def add_plain(self, a, pt): return self._plain("evab_add_plain", a, pt)
    def sub_plain(self, a, pt): return self._plain("evab_sub_plain", a, pt)
    def mul_plain(self, a, pt): return self._plain("evab_mul_plain", a, pt)

    def sum_terms(self, cts, pts):
        n = len(cts)
        ell = cts[0].shape[1]
        shape = (max(c.shape[0] for c in cts), ell, self.N)
        dc = [self._up(c) for c in cts]
        dp = [self._up(p) if p is not None else None for p in pts]
        do = self._alloc(int(np.prod(shape)) * 8)
        cp = (C.c_void_p * n)(*[d.value for d in dc])
        pp = (C.c_void_p * n)(*[(d.value if d is not None else None) for d in dp])
        sz = (C.c_int * n)(*[c.shape[0] for c in cts])
        self._chk(self.lib.evab_sum_terms(self.h, ell, do, n, cp, sz, pp, None))
        out = self._down(do, shape)
        self._free(do, *dc, *[d for d in dp if d is not None])
        return out

    def sum_products(self, cts, seconds, kinds):
        n = len(cts)
        ell = cts[0].shape[1]
        sout = max(3 if k == 2 else c.shape[0] for c, k in zip(cts, kinds))
        shape = (sout, ell, self.N)
        dc = [self._up(c) for c in cts]
        dp = [self._up(p) if p is not None else None for p in seconds]
        do = self._alloc(int(np.prod(shape)) * 8)
        cp = (C.c_void_p * n)(*[d.value for d in dc])
        pp = (C.c_void_p * n)(*[(d.value if d is not None else None) for d in dp])
        sz = (C.c_int * n)(*[c.shape[0] for c in cts])
        kd = (C.c_int * n)(*kinds)
        self._chk(self.lib.evab_sum_products(self.h, ell, do, n, cp, sz, pp, kd, None))
        out = self._down(do, shape)
        self._free(do, *dc, *[d for d in dp if d is not None])
        return out

    def negate(self, a):
        da, do = self._up(a), self._alloc(a.nbytes)
        self._chk(self.lib.evab_negate(self.h, a.shape[1], do, da, a.shape[0], None))
        out = self._down(do, a.shape)
        self._free(da, do)
        return out

    def mul(self, a, b):
        shape = (3, a.shape[1], self.N)
        da, db, do = self._up(a), self._up(b), self._alloc(int(np.prod(shape)) * 8)
        self._chk(self.lib.evab_mul(self.h, a.shape[1], do, da, db, None))
        out = self._down(do, shape)
        self._free(da, db, do)
        return out

    def square(self, a):
        shape = (3, a.shape[1], self.N)
        da, do = self._up(a), self._alloc(int(np.prod(shape)) * 8)
        self._chk(self.lib.evab_square(self.h, a.shape[1], do, da, None))
        out = self._down(do, shape)
        self._free(da, do)
        return out

    def rescale(self, a):
        shape = (a.shape[0], a.shape[1] - 1, self.N)
        da, do = self._up(a), self._alloc(int(np.prod(shape)) * 8)
        dw = self._alloc(self.lib.evab_rescale_work_bytes(self.h, a.shape[0]))
        self._chk(self.lib.evab_rescale(self.h, a.shape[1], do, da, a.shape[0], dw, None))
        out = self._down(do, shape)
        self._free(da, do, dw)
        return out

    def mod_switch(self, a):
        shape = (a.shape[0], a.shape[1] - 1, self.N)
        da, do = self._up(a), self._alloc(int(np.prod(shape)) * 8)
        self._chk(self.lib.evab_mod_switch(self.h, a.shape[1], do, da, a.shape[0], None))
        out = self._down(do, shape)
        self._free(da, do)
        return out

    def relinearize(self, a, rk):
        shape = (2, a.shape[1], self.N)
        da, dk, do = self._up(a), self._up(rk), self._alloc(int(np.prod(shape)) * 8)
        dw = self._alloc(self.lib.evab_keyswitch_work_bytes(self.h, a.shape[1]))
        self._chk(self.lib.evab_relinearize(self.h, a.shape[1], do, da, dk, dw, None))
        out = self._down(do, shape)
        self._free(da, dk, do, dw)
        return out

    def encode_uniform(self, values, scale, ell):
        n = len(values)
        vals = (C.c_double * n)(*[float(v) for v in values])
        scales = (C.c_double * n)(*([float(scale)] * n))
        do = self._alloc(n * ell * self.N * 8)
        self._chk(self.lib.evab_encode_uniform(self.h, n, vals, scales, ell, do, None))
        out = self._down(do, (n, ell, self.N))
        self._free(do)
        return out

    def rotate_many(self, a, steps_list, gks):
        ell = a.shape[1]
        da = self._up(a)
        dh = self._alloc(ell * self.N * 8)
        self._chk(self.lib.evab_rotate_prepare(self.h, ell, dh, da, None))
        outs = []
        for s_, gk in zip(steps_list, gks):
            elt = _elt(self.N, s_)
            if elt not in self._prepared:
                self._chk(self.lib.evab_galois_prepare(self.h, C.c_uint64(elt)))
                self._prepared.add(elt)
            dk, do = self._up(gk), self._alloc(2 * ell * self.N * 8)
            dw = self._alloc(self.lib.evab_keyswitch_work_bytes(self.h, ell))
            self._chk(self.lib.evab_rotate_prepared(self.h, ell, do, da, dh, C.c_uint64(elt), dk, dw, None))
            outs.append(self._down(do, (2, ell, self.N)))
            self._free(dk, do, dw)
        self._free(da, dh)
        return outs

    def decode(self, pt, scale, primes=None):
        lib = self.lib
        ell = pt.shape[0]
        dp = self._up(pt)
        do = self._alloc(self.N // 2 * 8)
        dw = self._alloc(lib.evab_decode_work_bytes(self.h, ell))
        self._chk(lib.evab_decode(self.h, ell, dp, C.c_double(scale), do, dw, None))
        out = self._down(do, (self.N // 2,)).view(np.float64)
        self._free(dp, do, dw)
        return out

    def rotate_many_modup(self, a, steps_list, gks):
        """rotations of one ciphertext sharing inverse NTT AND mod-up (evab_rotate_modup_*): (outputs, zero flag)"""
        lib = self.lib
        ell = a.shape[1]
        da = self._up(a)
        that = self._alloc(ell * self.N * 8)
        ext = self._alloc(lib.evab_rotate_modup_ext_bytes(self.h, ell))
        zf = self._alloc(8)
        self._chk(lib.evab_memset_zero(self.h, zf, 8, None))
        self._chk(lib.evab_rotate_modup_prepare(self.h, ell, that, ext, da, zf, None))
        work = self._alloc(lib.evab_rotate_modup_work_bytes(self.h, ell))
        outs, elts, dks, dcs = [], [], [], []
        for s_, gk in zip(steps_list, gks):
            elt = _elt(self.N, s_)
            if elt not in self._prepared:
                self._chk(lib.evab_galois_prepare(self.h, C.c_uint64(elt)))
                self._prepared.add(elt)
            dk = self._up(gk)
            cadd = self._alloc(lib.evab_hoist_const_bytes(self.h, ell))
            tmp = self._alloc((ell + 1) * self.N * 8)
            self._chk(lib.evab_rotate_hoist_const(self.h, ell, C.c_uint64(elt), dk, cadd, tmp, None))
            do = self._alloc(2 * ell * self.N * 8)
            self._chk(lib.evab_rotate_modup_prepared(self.h, ell, do, da, ext, C.c_uint64(elt), dk, cadd, work, None))
            outs.append(self._down(do, (2, ell, self.N)))
            self._free(do, tmp)
            elts.append(elt); dks.append(dk); dcs.append(cadd)
        # the same rotations in one call (evab_rotate_modup_many)
        n = len(steps_list)
        self._chk(lib.evab_rotate_modup_scale_c0(self.h, ell, ext, da, None))
        mw = self._alloc(lib.evab_rotate_modup_many_work_bytes(self.h, ell, n))
        dm = self._alloc(n * 2 * ell * self.N * 8)
        self._chk(lib.evab_rotate_modup_many(self.h, ell, n, dm, da, ext, (C.c_uint64 * n)(*elts), (C.c_void_p * n)(*dks), (C.c_void_p * n)(*dcs), mw, None))
        many = self._down(dm, (n, 2, ell, self.N))
        self.many = [many[i] for i in range(n)]
        flag = int(self._down(zf, (1,))[0])
        self._free(da, that, ext, work, zf, mw, dm, *dks, *dcs)
        return outs, flag

    def rotate(self, a, steps, gk):
        elt = int(self.lib.evab_galois_elt_from_step(C.c_uint64(self.N), steps))
        assert elt == _elt(self.N, steps)
        if elt not in self._prepared:
            self._chk(self.lib.evab_galois_prepare(self.h, C.c_uint64(elt)))
            self._prepared.add(elt)
        shape = (2, a.shape[1], self.N)
        da, dk, do = self._up(a), self._up(gk), self._alloc(int(np.prod(shape)) * 8)
        dw = self._alloc(self.lib.evab_keyswitch_work_bytes(self.h, a.shape[1]))
        self._chk(self.lib.evab_rotate(self.h, a.shape[1], do, da, C.c_uint64(elt), dk, dw, None))
        out = self._down(do, shape)
        self._free(da, dk, do, dw)
        return out

    def lazy_rotsum(self, a, steps_list, gks, weight_sets, scale):
        lib = self.lib
        ell = a.shape[1]
        da = self._up(a)
        that = self._alloc(ell * self.N * 8)
        ext = self._alloc(lib.evab_rotate_modup_ext_bytes(self.h, ell))
        zf = self._alloc(8)
        self._chk(lib.evab_memset_zero(self.h, zf, 8, None))
        self._chk(lib.evab_rotate_modup_prepare(self.h, ell, that, ext, da, zf, None))
        self._chk(lib.evab_rotate_modup_scale_c0(self.h, ell, ext, da, None))
        n, nout = len(steps_list), len(weight_sets)
        where = [(o, i) for o in range(nout) for i in range(n) if weight_sets[o][i] is not None]
        vecs = [np.ascontiguousarray(weight_sets[o][i], dtype=np.float64) for o, i in where]
        m = len(vecs)
        dv = [self._up(v.view(np.uint64)) for v in vecs]
        ptrs = (C.c_void_p * m)(*dv)
        sizes = (C.c_uint32 * m)(*[len(v) for v in vecs])
        scales = (C.c_double * m)(*([float(scale)] * m))
        dpts = self._alloc(m * (ell + 1) * self.N * 8)
        dw = self._alloc(lib.evab_encode_work_bytes(self.h, m))
        self._chk(lib.evab_encode_ext(self.h, m, ptrs, sizes, scales, ell, 1, dpts, dw, None))
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
        stride = (ell + 1) * self.N * 8
        wl = [None] * (nout * n)
        for idx, (o, i) in enumerate(where):
            wl[o * n + i] = dpts.value + idx * stride
        wts = (C.c_void_p * (nout * n))(*wl)
        work = self._alloc(lib.evab_lazy_rotsum_work_bytes(self.h, ell, nout))
        do = self._alloc(nout * 2 * ell * self.N * 8)
        self._chk(lib.evab_lazy_rotsum(self.h, ell, nout, do, da, ext, n, (C.c_uint64 * n)(*elts), (C.c_void_p * n)(*dks), (C.c_void_p * n)(*dcs), wts, work, None))
        out = self._down(do, (nout, 2, ell, self.N))
        pts = self._down(dpts, (m, ell + 1, self.N))
        flag = int(self._down(zf, (1,))[0])
        self._free(da, that, ext, zf, dpts, dw, work, do, *dv, *dks, *dcs)
        return out, {oi: pts[idx] for idx, oi in enumerate(where)}, flag
