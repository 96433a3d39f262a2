"""Seed-compressed evaluation keys on the GPU: evab_expand_key_uniform against the CPU replay and the numpy rule, keys from
generate_keys (c1 = the expansion of their seeds, valid key-switch keys), and B200Server / serialization with compressed keys
giving the same bytes as with the same keys in full."""
import ctypes as C

import numpy as np
import pytest

from backends import GpuBackend
from oracle import oracle as o
from test_compressed_keys import HIGH_REJECTION, np_expand, replay, seeds_for

pytestmark = pytest.mark.gpu


def device_expand(N, primes, moduli, seeds):
    be = GpuBackend(N, primes)
    k, n = len(primes), len(seeds)
    shape = (n, k - 1, 2, k, N)
    keys = np.full(shape, 0xDEADBEEF, dtype=np.uint64)
    dk = be._up(keys)
    ds = be._up(np.frombuffer(b"".join(seeds), dtype=np.uint64))
    qa = np.array(moduli, dtype=np.uint64)
    be._chk(be.lib.evab_expand_key_uniform(be.h, n, ds, qa.ctypes.data_as(C.POINTER(C.c_uint64)), dk, None))
    got = be._down(dk, shape)
    be.lib.evab_free(be.h, dk, None)
    be.lib.evab_free(be.h, ds, None)
    assert (got[:, :, 0] == 0xDEADBEEF).all()
    return got


@pytest.mark.parametrize("N,bits", [(16384, [60] * 5), (32768, [60] * 14)])
def test_device_expansion_equals_replay(N, bits):
    primes = o.gen_primes(N, bits)
    seeds = seeds_for(3, N)
    got = device_expand(N, primes, primes, seeds)
    assert np.array_equal(got, replay(seeds, N, primes))
    if len(bits) == 5:
        assert np.array_equal(got[0, :, 1], np_expand(seeds[0], N, primes)[0])


def test_device_expansion_high_rejection_moduli():
    N = 16384
    primes = o.gen_primes(N, [60] * 3)
    seeds = seeds_for(2, 9)
    got = device_expand(N, primes, HIGH_REJECTION, seeds)
    assert np.array_equal(got, replay(seeds, N, HIGH_REJECTION))
    want, fell = np_expand(seeds[1], N, HIGH_REJECTION)
    assert (fell > 0).all() and np.array_equal(got[1, :, 1], want)


def test_device_expansion_rejects_bad_arguments():
    primes = o.gen_primes(1024, [60] * 3)
    be = GpuBackend(1024, primes)
    qa = np.array(primes, dtype=np.uint64)
    for n in (0, 65536):
        assert be.lib.evab_expand_key_uniform(be.h, n, None, qa.ctypes.data_as(C.POINTER(C.c_uint64)), None, None) != 0
    qa[1] = 1
    assert be.lib.evab_expand_key_uniform(be.h, 1, None, qa.ctypes.data_as(C.POINTER(C.c_uint64)), None, None) != 0
    assert b"modulus" in be.lib.evab_last_error()


# ---------------------------------------------------------------------------------------------------- keys from generate_keys
def _bitrev(N):
    logn = N.bit_length() - 1
    return np.array([int(format(i, "0%db" % logn)[::-1], 2) for i in range(N)], dtype=np.int64)


def _mulmod(a, b, q):
    return (a.astype(object) * b.astype(object) % q).astype(np.uint64)


def _check_key(key, s, s_new, primes, orc):
    """digit J: c0 + c1 s - P [J] s' is a small error (taken back to coefficients with the oracle's NTT)"""
    k, P = len(primes), primes[-1]
    for J in range(k - 1):
        for m in range(k):
            q = primes[m]
            v = (key[J, 0, m].astype(object) + _mulmod(key[J, 1, m], s[m], q).astype(object)) % q
            if m == J:
                v = (v - (P % q) * s_new[m].astype(object)) % q
            e = orc.ntt_inv(np.array(v, dtype=np.uint64), m).astype(object)
            e = np.where(e > q // 2, e - q, e)
            assert max(abs(int(x)) for x in e) <= 42, (J, m)


def test_generated_keys_are_their_seeds_expansion_and_valid():
    from eva_b200 import b200, program_io as gl
    from eva_b200.ckks import CKKSParameters
    _, params, _, _ = gl.build_program(gl.load_json("polynomial"))
    params = CKKSParameters(list(params.prime_bits), {1, -3}, params.poly_modulus_degree)
    pub, sec = b200.generate_keys(params, seed=5)
    x = pub._export()
    sk = sec._export()["secret_key"]
    N, primes = x["N"], list(x["primes"])
    k = len(primes)
    assert isinstance(x["relin_seed"], bytes) and len(x["relin_seed"]) == 32
    assert sorted(x["galois_seeds"]) == sorted(x["galois_keys"])
    elts = sorted(x["galois_keys"])
    keys = [x["relin_key"]] + [x["galois_keys"][e] for e in elts]
    seeds = [x["relin_seed"]] + [x["galois_seeds"][e] for e in elts]
    exp = replay(seeds, N, primes)
    for g, key in enumerate(keys):
        assert np.array_equal(key[:, 1], exp[g, :, 1]), g
    orc = o.Oracle(N, primes=primes)
    s2 = np.stack([_mulmod(sk[m], sk[m], primes[m]) for m in range(k)])
    _check_key(x["relin_key"], sk, s2, primes, orc)
    br = _bitrev(N)
    for e in elts:
        src = br[((e * (2 * br + 1)) >> 1) & (N - 1)]
        _check_key(x["galois_keys"][e], sk, sk[:, src], primes, orc)
    # the same seed gives the same keys and seeds; the public key is drawn before them
    again = b200.generate_keys(params, seed=5)[0]._export()
    assert again["relin_seed"] == x["relin_seed"] and np.array_equal(again["public_key"], x["public_key"])


# ------------------------------------------------------------------------------------------------ servers: compressed == full
CLIENT_SEEDS = (11, 12, 13)


class Clients:
    """a golden program and three clients' generate_keys contexts; ciphertext inputs made with an oracle on the same primes"""

    def __init__(self, name):
        from eva_b200 import b200, program_io as gl
        self.d = d = gl.load_json(name)
        self.prog, self.params, _, _ = gl.build_program(d)
        self.pubs = [b200.generate_keys(self.params, seed=s)[0] for s in CLIENT_SEEDS]
        self.full = [(p._export()["relin_key"], dict(p._export()["galois_keys"])) for p in self.pubs]
        orc = o.Oracle(d["poly_modulus_degree"], d["prime_bits"]).keygen(1)
        self.vals = []
        for i in range(4):
            rng = np.random.default_rng(60 + i)
            val = b200.B200Valuation()
            for name_, info in d["signature"].items():
                x = rng.uniform(0.0, 0.2, d["vec_size"])
                ell, scale = orc.k - 1 - info["level"], 2.0 ** info["scale"]
                if info["type"] == "Cipher":
                    val.set_cipher(name_, orc.encrypt(orc.encode(x, scale, ell), seed=60 + i), scale)
                elif info["type"] == "Raw":
                    val.set_raw(name_, list(x))
                else:
                    val.set_plain(name_, orc.encode(x, scale, ell), scale)
            self.vals.append(val)

    def run(self, server, assign):
        outs = server.execute_batch(self.prog, list(zip(assign, self.vals)))
        return [{n: out.get(n) for n in self.d["outputs"]} for out in outs]


def _same(a, b, what):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        for n in x:
            kx, ky = x[n][0], y[n][0]
            assert kx == ky, (what, i, n)
            if kx == "cipher":
                assert np.array_equal(x[n][1], y[n][1]) and x[n][2] == y[n][2], (what, i, n)
            else:
                assert np.array_equal(np.asarray(x[n][1]), np.asarray(y[n][1])), (what, i, n)


@pytest.mark.parametrize("name", ["sobel", "harris", "feat_mixed"])
def test_compressed_and_full_servers_give_the_same_bytes(name):
    from eva_b200 import b200
    c = Clients(name)
    full = b200.B200Server(c.params, capacity=3)
    comp = b200.B200Server(c.params, capacity=3)
    for t, p in enumerate(c.pubs):
        assert full.add_raw_keys(*c.full[t]) == t
        assert comp.add_keys(p) == t
    info = comp.bank_info()
    assert info["compressed_tenants"] == 3 and full.bank_info()["compressed_tenants"] == 0
    batches = [[0, 1, 2, 0], [2, 2, 1, 0], [1, 0, 2, 1]]
    want = [c.run(full, a) for a in batches]
    for a, w in zip(batches, want):
        _same(c.run(comp, a), w, (name, "resident", a))
    # paging: 2 slots, compressed tenants evicted and filled again
    paged = b200.B200Server(c.params, capacity=2, max_tenants=4)
    for p in c.pubs:
        paged.add_keys(p)
    for a in ([2, 2, 2, 2], [0, 1, 0, 1], [1, 2, 2, 1], [0, 0, 0, 0], [2, 0, 0, 2]):
        _same(c.run(paged, a), c.run(full, a), (name, "paged", a))
    pi = paged.bank_info()
    assert pi["evictions"] > 0 and pi["fills"] > 3 and pi["compressed_tenants"] == 3
    # one server holding both forms of the same clients (tenant t compressed, t + 3 full), mixed in one batch
    mixed = b200.B200Server(c.params, capacity=2, max_tenants=6)
    for p in c.pubs:
        mixed.add_keys(p)
    for t in range(3):
        assert mixed.add_raw_keys(*c.full[t]) == 3 + t
    _same(c.run(mixed, [0, 4, 0, 4]), c.run(full, [0, 1, 0, 1]), (name, "mixed"))
    _same(c.run(mixed, [5, 2, 2, 5]), c.run(full, [2, 2, 2, 2]), (name, "mixed same client"))
    _same(c.run(mixed, [3, 1, 1, 3]), c.run(full, [0, 1, 1, 0]), (name, "mixed refill"))
    # host store: the exact compressed size for compressed tenants, the full size for full ones
    k, N, keys = len(c.params.prime_bits), c.d["poly_modulus_degree"], 1 + len(pi["galois_elements"])
    comp_bytes = keys * ((k - 1) * k * N * 8 + 32)
    full_bytes = keys * (k - 1) * 2 * k * N * 8
    assert pi["host_key_bytes"] == 3 * comp_bytes
    mi = mixed.bank_info()
    assert mi["host_key_bytes"] == 3 * comp_bytes + 3 * full_bytes and mi["compressed_tenants"] == 3
    if name == "sobel":
        assert comp_bytes == 26214400 + 320 and full_bytes == 52428800


def test_add_compressed_keys_directly_and_errors():
    from eva_b200 import b200
    c = Clients("polynomial")
    x = c.pubs[0]._export()
    rc0 = np.ascontiguousarray(x["relin_key"][:, 0])
    gc0 = {e: np.ascontiguousarray(v[:, 0]) for e, v in x["galois_keys"].items()}
    s = b200.B200Server(c.params, capacity=2)
    elts = s.bank_info()["galois_elements"]
    full = b200.B200Server(c.params, capacity=1)
    full.add_raw_keys(*c.full[0])
    assert s.add_compressed_keys(rc0, x["relin_seed"], gc0, x["galois_seeds"]) == 0
    _same(c.run(s, [0, 0, 0, 0]), c.run(full, [0, 0, 0, 0]), "direct")
    with pytest.raises(Exception, match="32 bytes"):
        s.add_compressed_keys(rc0, x["relin_seed"][:31], gc0, x["galois_seeds"])
    if elts:
        bad = dict(x["galois_seeds"]); bad[elts[0]] = b"\0" * 33
        with pytest.raises(Exception, match="32 bytes"):
            s.add_compressed_keys(rc0, x["relin_seed"], gc0, bad)
        missing = {e: v for e, v in gc0.items() if e != elts[0]}
        with pytest.raises(Exception, match="missing"):
            s.add_compressed_keys(rc0, x["relin_seed"], missing, x["galois_seeds"])
    with pytest.raises(Exception, match="does not match"):
        s.add_compressed_keys(np.ascontiguousarray(rc0[:, :-1]), x["relin_seed"], gc0, x["galois_seeds"])
    with pytest.raises(Exception, match="does not match"):
        s.add_compressed_keys(x["relin_key"], x["relin_seed"], gc0, x["galois_seeds"])      # full shape where c0 rows are expected
    from eva_b200.ckks import CKKSParameters
    other, _ = b200.generate_keys(CKKSParameters([40] + list(c.params.prime_bits)[1:], c.params.rotations, c.params.poly_modulus_degree), seed=3)
    with pytest.raises(Exception, match="N / primes"):
        s.add_keys(other)
    assert s.bank_info()["tenants"] == 1 and s.bank_info()["compressed_tenants"] == 1


def test_saved_compressed_context_is_half_and_loads_bit_identically():
    from eva_b200 import b200, serialization as ser
    c = Clients("sobel")
    pub = c.pubs[0]
    blob = ser.dumps(pub)
    x = pub._export()
    full_ctx = b200.public_from_raw(x["N"], x["primes"], x["public_key"], x["relin_key"], dict(x["galois_keys"]))
    full_blob = ser.dumps(full_ctx)
    assert "relin_seed" not in full_ctx._export()
    keys = 1 + len(x["galois_keys"])
    assert 0.45 < len(blob) / len(full_blob) < 0.55, (len(blob), len(full_blob))
    assert len(full_blob) - len(blob) >= keys * x["relin_key"].nbytes // 2 - keys * 64
    loaded = ser.loads(blob)
    y = loaded._export()
    assert y["relin_seed"] == x["relin_seed"] and y["galois_seeds"] == x["galois_seeds"]
    assert np.array_equal(y["relin_key"], x["relin_key"]) and np.array_equal(y["public_key"], x["public_key"])
    for e in x["galois_keys"]:
        assert np.array_equal(y["galois_keys"][e], x["galois_keys"][e])
    # execution through the loaded context equals the original's, byte for byte
    a, b = pub.execute(c.prog, c.vals[0]), loaded.execute(c.prog, c.vals[0])
    for n in c.d["outputs"]:
        assert np.array_equal(a.get(n)[1], b.get(n)[1])
    # full-format files still load, and a server takes the loaded compressed context compressed
    again = ser.loads(full_blob)
    assert "relin_seed" not in again._export() and np.array_equal(again._export()["relin_key"], x["relin_key"])
    s = b200.B200Server(c.params, capacity=2)
    assert (s.add_keys(loaded), s.add_keys(again)) == (0, 1)
    assert s.bank_info()["compressed_tenants"] == 1
    _same(c.run(s, [0, 1, 0, 1]), c.run(s, [1, 0, 1, 0]), "loaded compressed vs loaded full")
