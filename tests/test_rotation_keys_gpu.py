"""Rotations composed from power-of-two Galois keys, on the GPU: every result is bit-identical to the oracle's chained rotations
(SEAL's rotate_vector restated in test_rotation_keys.seal_hops, each hop one oracle rotation with the oracle's keys), on single
rotations, on every intermediate term of the workloads and fixture programs under every execution path and the options that
change how rotations run, and on B200Server tenants, resident and paged.  generate_keys(rotation_keys="power_of_two") keys meet
the reference's MSE criterion and survive save / load."""
import os

import numpy as np
import pytest

from oracle import oracle as o
from oracle_exec import OracleProgram
from test_rotation_keys import elements, power_of_two_steps, rotation_program, seal_hops

pytestmark = pytest.mark.gpu


class ComposedOracleProgram(OracleProgram):
    """the oracle runner with SEAL's rotate_vector over the keys of `steps`: a rotation without its own key is its chain of hops"""

    def __init__(self, d, orc, steps):
        super().__init__(d, orc)
        self.rk = orc.relin_key()
        self.gks = {o.galois_elt_from_step(orc.N, s): orc.galois_key(o.galois_elt_from_step(orc.N, s)) for s in steps}

    def exec_term(self, t, V):
        if t["op"] in ("RotateLeftConst", "RotateRightConst") and t["rotation"] != 0 and V[t["args"][0]][0] == "cipher":
            x = V[t["args"][0]]
            return ("cipher", chain_rotate(self.orc, x[1], t["rotation"] if t["op"] == "RotateLeftConst" else -t["rotation"], self.gks), x[2])
        return super().exec_term(t, V)


def chain_rotate(orc, ct, steps, gks):
    for h in seal_hops(orc.N, steps, set(gks)):
        ct = orc.rotate(ct, h, gks[o.galois_elt_from_step(orc.N, h)])
    return ct


def public_with(orc, steps):
    from eva_b200 import b200
    return b200.context_from_raw_keys(orc.N, orc.primes, orc.relin_key(),
                                      {o.galois_elt_from_step(orc.N, s): orc.galois_key(o.galois_elt_from_step(orc.N, s)) for s in steps})


# ---------------------------------------------------------------------------------------------------------------------------
# single rotations

def _single(orc, steps, keys):
    from eva_b200 import b200
    N = orc.N
    prog, x, terms = rotation_program(N, steps)
    pub = public_with(orc, keys)
    ct = orc.encrypt(orc.encode(np.random.default_rng(3).uniform(-1, 1, N // 2), 2.0 ** 30, orc.k - 1), seed=5)
    val = b200.B200Valuation()
    val.set_cipher("x", ct, 2.0 ** 30)
    gks = {o.galois_elt_from_step(N, s): orc.galois_key(o.galois_elt_from_step(N, s)) for s in keys}
    for opts in ({}, dict(hoist_mod_up=False), dict(rotation_chunk=1), dict(hoist_rotations=False)):
        pub.set_options(**opts)
        out = pub.execute(prog, val)
        for s in steps:
            assert np.array_equal(out.get("r%d" % s)[1], chain_rotate(orc, ct, s, gks)), (s, opts)
    return pub, prog


def test_single_rotations_direct_composed_and_half_ring_edge():
    """3, -3, 7, 63, 129 composed; N/2 - 1 and 3N/8 by the keys of -1 and -N/8 (their NAF's N/2 term dropped); vec_size N/2"""
    orc = o.Oracle(4096, [60, 60, 60]).keygen(2)
    N = orc.N
    steps = [3, -3, 7, 63, 129, N // 2 - 1, 3 * N // 8]
    keys = power_of_two_steps(N, steps)
    assert keys == [-N // 8, -4, -1, 1, 4, 8, 64, 128]
    pub, prog = _single(orc, steps, keys)
    st = pub.plan_stats(prog)
    assert st["composed_rotations"] == 5


def test_single_rotations_mixed_key_prefix():
    """keys {-1, -4, 16, -5}: rot_-5 by its own key, rot_11 = rot_16(rot_-4(rot_-1(x))) -- never through rot_-5"""
    orc = o.Oracle(4096, [60, 60, 60]).keygen(4)
    pub, prog = _single(orc, [-5, -1, 11, -4], [-1, -4, 16, -5])
    assert pub.plan_stats(prog)["composed_rotations"] == 1


# ---------------------------------------------------------------------------------------------------------------------------
# every intermediate term of the workloads and fixture programs

NAMES = ["sobel", "harris", "wide64", "feat_rot_0", "feat_rot_1", "feat_rot_m1", "feat_rot_m2", "feat_hsum", "feat_mixed"]
OPTIONS = {"default": {}, "no_hoist_mod_up": dict(hoist_mod_up=False), "chunk1": dict(rotation_chunk=1),
           "no_rotation_sums": dict(rotation_sums=False)}
DISTINCT = 4
BATCH = 32


class Fixture:
    """a program, oracle keys of seed 1 restricted to the power-of-two set, DISTINCT valuations and their oracle values"""

    def __init__(self, name):
        from eva_b200 import b200, program_io as gl
        from eva_b200._eva_b200 import _rotation_key_steps
        self.d = d = gl.load_json(name)
        self.prog, self.params, self.sig, self.terms = gl.build_program(d)
        self.N = N = d["poly_modulus_degree"]
        self.orc = orc = o.Oracle(N, d["prime_bits"]).keygen(1)
        self.keys = _rotation_key_steps(self.params, "power_of_two")
        assert self.keys == power_of_two_steps(N, d["rotations"])
        self.op = ComposedOracleProgram(d, orc, self.keys)
        self.pub = public_with(orc, self.keys)
        self.vals, self.ins, self.want = [], [], []
        for i in range(DISTINCT):
            rng = np.random.default_rng(20 + i)
            val, io = b200.B200Valuation(), {}
            for name_, info in d["signature"].items():
                x = rng.uniform(0.0, 0.2, d["vec_size"])
                ell, scale = orc.k - 1 - info["level"], 2.0 ** info["scale"]
                if info["type"] == "Cipher":
                    ct = orc.encrypt(orc.encode(x, scale, ell), seed=30 + i)
                    val.set_cipher(name_, ct, scale); io[name_] = ("cipher", ct, scale)
                elif info["type"] == "Raw":
                    val.set_raw(name_, list(x)); io[name_] = ("raw", x)
                else:
                    pt = orc.encode(x, scale, ell)
                    val.set_plain(name_, pt, scale); io[name_] = ("plain", pt, scale)
            self.vals.append(val); self.ins.append(io)
            self.want.append(self.op.run(io))

    def check_outputs(self, out, i, what):
        for oname, oid in self.d["outputs"].items():
            kind, arr, scale = out.get(oname)
            want = self.want[i][oid]
            if kind == "cipher":
                assert np.array_equal(arr, want[1]) and scale == want[2], (what, i, oname)

    def check_terms(self, batch, b, i, what):
        """every materialised term of instance b (valuation i) through debug_value"""
        checked = 0
        for t in self.d["terms"]:
            want = self.want[i][t["id"]]
            if want[0] != "cipher":
                continue
            got = self.pub.debug_value(self.prog, self.terms[t["id"]].index, batch, b)
            if got is None:          # fused away
                continue
            assert np.array_equal(got[0], want[1]) and got[1] == want[2], (what, b, t["id"], t["op"])
            checked += 1
        return checked


_FIX = {}


def fixture(name):
    if name not in _FIX:
        _FIX[name] = Fixture(name)
    return _FIX[name]


@pytest.mark.parametrize("option", sorted(OPTIONS))
@pytest.mark.parametrize("name", NAMES)
def test_every_term_exact(name, option):
    """execute, execute_batch (32 instances, one plan) and execute_batch_async: every output and every materialised intermediate
    equals the oracle's chained rotations"""
    f = fixture(name)
    opts = OPTIONS[option]
    f.pub.set_options(**opts)
    f.check_outputs(f.pub.execute(f.prog, f.vals[0]), 0, "execute")
    rot = sum(1 for t in f.d["terms"] if t["op"].startswith("Rotate") and t["rotation"])
    assert f.check_terms(1, 0, 0, "execute") > 0 or rot == 0
    assign = [b % DISTINCT for b in range(BATCH)]
    f.pub.set_options(fuse=BATCH, **opts)
    outs = f.pub.execute_batch(f.prog, [f.vals[i] for i in assign])
    for b, i in enumerate(assign):
        f.check_outputs(outs[b], i, "execute_batch")
    for b in (0, 1, 2, 3, BATCH - 1):
        f.check_terms(BATCH, b, assign[b], "execute_batch")
    f.pub.set_options(fuse=8, **opts)
    h0 = f.pub.execute_batch_async(f.prog, [f.vals[i] for i in assign], 0)
    h1 = f.pub.execute_batch_async(f.prog, [f.vals[i] for i in assign[::-1]], 1)
    for h, a in ((h0, assign), (h1, assign[::-1])):
        for b, out in enumerate(f.pub.execute_batch_result(h)):
            f.check_outputs(out, a[b], "execute_batch_async")
    keyless = [s for s in f.params.rotations if s and o.galois_elt_from_step(f.N, s) not in elements(f.N, f.keys)]
    if keyless and option == "default":
        assert f.pub.plan_stats(f.prog)["composed_rotations"] > 0


def test_zero_digit_redo_with_chains():
    """an input with a zero digit coefficient: the run is redone without the shared mod-up, and the chains still give SEAL's bits"""
    from eva_b200 import b200
    f = fixture("sobel")
    pub = public_with(f.orc, f.keys)
    (name_, info), = f.d["signature"].items()
    ell = f.orc.k - 1 - info["level"]
    ct = f.orc.encrypt(f.orc.encode(np.random.default_rng(4).uniform(0, 0.2, f.d["vec_size"]), 2.0 ** info["scale"], ell), seed=3)
    c1 = np.stack([f.orc.ntt_inv(ct[1, r], r) for r in range(ell)])
    c1[1, 7] = 0
    ct[1] = np.stack([f.orc.ntt_fwd(c1[r], r) for r in range(ell)])
    val = b200.B200Valuation()
    val.set_cipher(name_, ct, 2.0 ** info["scale"])
    want = f.op.run({name_: ("cipher", ct, 2.0 ** info["scale"])})
    for _ in range(2):
        out = pub.execute(f.prog, val)
        for oname, oid in f.d["outputs"].items():
            assert np.array_equal(out.get(oname)[1], want[oid][1])


# ---------------------------------------------------------------------------------------------------------------------------
# B200Server with power-of-two key banks

def _host_bytes(info, k, N, full, compressed):
    keys = 1 + len(info["galois_elements"])
    return full * keys * (k - 1) * 2 * k * N * 8 + compressed * (keys * (k - 1) * k * N * 8 + 32 * keys)


@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_server_power_of_two_resident_and_paged(name):
    from eva_b200 import b200
    f = fixture(name)
    N, k = f.N, f.orc.k
    # tenants 0, 1: oracle keys (seeds 1 and 2); tenants 2, 3: generated power-of-two keys (compressed)
    orcs = [f.orc, o.Oracle(N, f.d["prime_bits"]).keygen(2)]
    ops = [f.op, ComposedOracleProgram(f.d, orcs[1], f.keys)]
    raw = [(x.relin_key(), {o.galois_elt_from_step(N, s): x.galois_key(o.galois_elt_from_step(N, s)) for s in f.keys}) for x in orcs]
    gen = [b200.generate_keys(f.params, rotation_keys="power_of_two")[0] for _ in range(2)]
    for capacity, max_tenants in ((4, None), (2, 5)):
        s = b200.B200Server(f.params, capacity=capacity, max_tenants=max_tenants, rotation_keys="power_of_two")
        info = s.bank_info()
        assert info["rotation_keys"] == "power_of_two"
        assert sorted(info["galois_elements"]) == sorted(elements(N, f.keys))
        assert [s.add_raw_keys(*r) for r in raw] == [0, 1]
        assert [s.add_keys(g) for g in gen] == [2, 3]
        info = s.bank_info()
        assert info["compressed_tenants"] == 2
        assert info["host_key_bytes"] == (_host_bytes(info, k, N, 2, 2) if max_tenants else 0)
        for pair in ((0, 1), (2, 3), (1, 2), (3, 0)):   # two tenants per batch: with 2 slots every batch pages
            assign = [(pair[b % 2], b % DISTINCT) for b in range(4)]
            outs = s.execute_batch(f.prog, [(t, f.vals[i]) for t, i in assign])
            for (t, i), out in zip(assign, outs):
                if t < 2:
                    V = f.want[i] if t == 0 else ops[1].run(f.ins[i])
                    for oname, oid in f.d["outputs"].items():
                        assert np.array_equal(out.get(oname)[1], V[oid][1]), (capacity, t, i)
                else:
                    ref = gen[t - 2].execute(f.prog, f.vals[i])
                    for oname in f.d["outputs"]:
                        assert np.array_equal(out.get(oname)[1], ref.get(oname)[1]), (capacity, t, i)
        if max_tenants:
            assert s.bank_info()["evictions"] > 0
        assert s.plan_stats(f.prog)["composed_rotations"] > 0


def test_server_refuses_a_context_without_a_hop_key():
    """wide4096's program keys are 0..63 (no -1, no 64): a power-of-two server needs those keys and names the first missing element"""
    from eva_b200 import b200, program_io as gl
    d = gl.load_json("wide4096")
    _, params, _, _ = gl.build_program(d)
    N = d["poly_modulus_degree"]
    pub, _ = b200.generate_keys(params, rotation_keys="program")
    s = b200.B200Server(params, capacity=1, rotation_keys="power_of_two")
    missing = set(s.bank_info()["galois_elements"]) - set(pub._export()["galois_keys"])
    assert missing == elements(N, [-16, -8, -4, -2, -1, 64])
    with pytest.raises(ValueError, match="element %d of the server's rotation set is missing" % min(missing)):
        s.add_keys(pub)
    # the program-key server takes it, and a power-of-two context is refused by it (it lacks the key of 3, say)
    sp = b200.B200Server(params, capacity=1)
    assert sp.add_keys(pub) == 0
    p2, _ = b200.generate_keys(params, rotation_keys="power_of_two")
    with pytest.raises(ValueError, match="missing"):
        sp.add_keys(p2)


# ---------------------------------------------------------------------------------------------------------------------------
# generate_keys(rotation_keys="power_of_two")

GOLDEN = "image_processing_baboon.npz"


def _golden(name):
    import tests_programs
    from eva_b200.ckks import CKKSCompiler
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", GOLDEN))
    inputs = {"image": [x / 255.0 for x in g["image"].tolist()]}
    compiled, params, signature = CKKSCompiler().compile(getattr(tests_programs, name)())
    return compiled, params, signature, inputs, g[name]


@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_generated_power_of_two_keys_meet_the_reference_criterion(name, tmp_path):
    from eva_b200 import b200, load, save
    compiled, params, signature, inputs, expected = _golden(name)
    pub, sec = b200.generate_keys(params, rotation_keys="power_of_two")
    N = params.poly_modulus_degree
    assert sorted(pub._export()["galois_keys"]) == sorted(elements(N, power_of_two_steps(N, params.rotations)))
    enc = pub.encrypt(inputs, signature)
    res = pub.execute(compiled, enc)
    assert pub.plan_stats(compiled)["composed_rotations"] > 0
    assert np.mean((np.array(sec.decrypt(res, signature)["image"]) - expected) ** 2) < 0.01
    # approx_hoist with chains: graded by the same criterion
    pub.set_options(approx_hoist=True)
    assert np.mean((np.array(sec.decrypt(pub.execute(compiled, enc), signature)["image"]) - expected) ** 2) < 0.01
    pub.set_options()
    # save / load: the same key set, the same bytes
    save(pub, str(tmp_path / "p.sealpublic"))
    pub2 = load(str(tmp_path / "p.sealpublic"))
    assert sorted(pub2._export()["galois_keys"]) == sorted(pub._export()["galois_keys"])
    res2 = pub2.execute(compiled, enc)
    for oname in res.names():
        assert np.array_equal(res2.get(oname)[1], res.get(oname)[1])


def test_program_keys_unchanged_by_default():
    """rotation_keys="program" is today's key set, bit for bit under a test seed"""
    from eva_b200 import b200
    compiled, params, signature, inputs, _ = _golden("sobel")
    a = b200.generate_keys(params, seed=9)[0]._export()
    b = b200.generate_keys(params, seed=9, rotation_keys="program")[0]._export()
    assert sorted(a["galois_keys"]) == sorted(elements(params.poly_modulus_degree, params.rotations))
    for e in a["galois_keys"]:
        assert np.array_equal(a["galois_keys"][e], b["galois_keys"][e])
    assert np.array_equal(a["relin_key"], b["relin_key"])


def test_errors():
    from eva_b200 import b200
    compiled, params, signature, inputs, _ = _golden("sobel")
    with pytest.raises(ValueError, match="rotation_keys"):
        b200.generate_keys(params, rotation_keys="powers_of_two")
    with pytest.raises(ValueError, match="rotation_keys"):
        b200.B200Server(params, capacity=1, rotation_keys="")
    # keys of 1 and 4 only: naf(3) = [-1, 4] has no key for -1
    orc = o.Oracle(4096, [60, 60, 60]).keygen(1)
    prog, _, _ = rotation_program(orc.N, [3])
    pub = public_with(orc, [1, 4])
    val = b200.B200Valuation()
    val.set_cipher("x", orc.encrypt(orc.encode(np.zeros(orc.N // 2), 2.0 ** 30, orc.k - 1)), 2.0 ** 30)
    e = o.galois_elt_from_step(orc.N, -1)
    with pytest.raises(ValueError, match=r"Galois key not present.*rotation by 3 steps.*term -1 \(Galois element %d\)" % e):
        pub.execute(prog, val)
