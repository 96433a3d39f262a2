"""Slot packing without a GPU: pack_program / pack_inputs / unpack_outputs (eva_b200.ckks).  k instances of a compiled program run in
one packed program whose plaintext semantics are exactly the k separate runs; the packed program has the same terms, scales and
levels, rotation steps (r mod v) * k and interleaved constants; it round-trips through save / load; the planner gives it the same
plan shape and cost; and the errors name the values involved."""
import os

import numpy as np
import pytest

from eva_b200 import EvaProgram, Input, Output, Op, evaluate, program_io as gl, serialization as ser
from eva_b200._eva_b200 import _plan, _rotation_key_steps
from eva_b200.ckks import CKKSCompiler, pack_inputs, pack_program, unpack_outputs

from backends import _elt
from test_planner import check_plan

FEAT_BIN = sorted(f[:-5] for f in os.listdir(os.path.join(os.path.dirname(__file__), "golden", "programs")) if f.startswith("feat_bin_"))
SEMANTICS = ["polynomial", "sobel", "harris", "feat_hsum", "feat_rot_m1", "feat_rot_m2", "feat_mixed"] + FEAT_BIN


def load(name):
    d = gl.load_json(name)
    prog, params, sig, _ = gl.build_program(d)
    return d, prog, params, sig


def max_k(prog, params):
    return params.poly_modulus_degree // 2 // prog.vec_size


def ks_for(prog, params):
    """2, the largest k, and one in between when there is one"""
    top = max_k(prog, params)
    return sorted({2, top, max(2, top // 16)})


def valuations(sig, k, seed, short=True):
    """k valuations with distinct values; with `short`, odd instances give vectors of vec_size / 4 values (replicated by pack_inputs
    and by evaluate alike)"""
    rng = np.random.default_rng(seed)
    v = sig.vec_size
    out = []
    for b in range(k):
        n = v // 4 if short and b % 2 and v >= 4 else v
        out.append({name: rng.uniform(-1.0, 1.0, n) for name in sig.inputs})
    return out


def check_semantics(prog, sig, packed, psig, k, seed=1):
    vals = valuations(sig, k, seed)
    pin = pack_inputs(vals, sig, k)
    assert set(pin) == set(sig.inputs) and all(len(x) == psig.vec_size for x in pin.values())
    got = unpack_outputs(evaluate(packed, pin), k)
    assert len(got) == k
    for b in range(k):
        want = evaluate(prog, {n: list(x) for n, x in vals[b].items()})
        assert set(got[b]) == set(want)
        for name in want:
            assert np.array_equal(got[b][name], np.asarray(want[name])), (b, name)


@pytest.mark.parametrize("name", SEMANTICS)
def test_plaintext_semantics_exact(name):
    _, prog, params, sig = load(name)
    for k in ks_for(prog, params):
        packed, pparams, psig = pack_program(prog, params, sig, k)
        check_semantics(prog, sig, packed, psig, k, seed=k)


def short_constant_program():
    """a program of vec_size 64 with dense constants of 4 and 16 values, a uniform constant, rotations both ways (one negative)
    and a Raw input"""
    p = EvaProgram("short_constants", vec_size=64)
    with p:
        x, w = Input("x"), Input("w", is_encrypted=False)
        y = (x << 3) * [0.5, -1.0, 2.0, 0.25] + (x >> 5) * [float(i) / 8 for i in range(16)]
        z = (y << -2) * 0.75 + w * [1.0, -2.0, 3.0, -4.0] + (x * x)
        Output("y", y)
        Output("z", z)
    p.set_output_ranges(20)
    p.set_input_scales(30)
    return CKKSCompiler({"warn_vec_size": "false"}).compile(p)


def test_constants_shorter_than_vec_size():
    prog, params, sig = short_constant_program()
    lens = sorted({len(t.attributes["ConstantValueAttribute"]) for t in prog.terms() if t.op == Op.Constant})
    assert 4 in lens and 16 in lens and 1 in lens
    for k in (2, 8, max_k(prog, params)):
        packed, pparams, psig = pack_program(prog, params, sig, k)
        check_semantics(prog, sig, packed, psig, k, seed=10 + k)
        plens = sorted({len(t.attributes["ConstantValueAttribute"]) for t in packed.terms() if t.op == Op.Constant})
        assert plens == sorted({1} | {n * k for n in lens if n > 1})


def check_structure(prog, params, sig, packed, pparams, psig, k):
    v = prog.vec_size
    assert packed.name == prog.name + ".pack%d" % k and packed.vec_size == v * k
    a, b = prog.terms(), packed.terms()
    assert len(a) == len(b)
    pos_a, pos_b = {t.index: i for i, t in enumerate(a)}, {t.index: i for i, t in enumerate(b)}
    steps = set()
    for s, t in zip(a, b):
        assert s.op == t.op
        assert [pos_a[o.index] for o in s.operands] == [pos_b[o.index] for o in t.operands]
        sa, ta = dict(s.attributes), dict(t.attributes)
        if s.op in (Op.RotateLeftConst, Op.RotateRightConst):
            r = sa.pop("RotationAttribute")
            step = ta.pop("RotationAttribute")
            assert step == (r % v) * k
            steps.add(step if s.op == Op.RotateLeftConst else -step)
        if s.op == Op.Constant:
            c = np.asarray(sa.pop("ConstantValueAttribute"))
            pc = np.asarray(ta.pop("ConstantValueAttribute"))
            if len(c) == 1:
                assert np.array_equal(pc, c)
            else:
                assert len(pc) == len(c) * k
                for j in range(k):
                    assert np.array_equal(pc[j::k], c)
        assert sa == ta   # type, scale, level, rescale divisor, range
    assert {n: pos_a[t.index] for n, t in prog.inputs.items()} == {n: pos_b[t.index] for n, t in packed.inputs.items()}
    assert {n: pos_a[t.index] for n, t in prog.outputs.items()} == {n: pos_b[t.index] for n, t in packed.outputs.items()}
    assert list(pparams.prime_bits) == list(params.prime_bits) and pparams.poly_modulus_degree == params.poly_modulus_degree
    assert pparams.rotations == steps   # every rotation of these programs is a ciphertext rotation
    assert psig.vec_size == v * k and set(psig.inputs) == set(sig.inputs)
    for n, e in sig.inputs.items():
        f = psig.inputs[n]
        assert (f.input_type, f.scale, f.level) == (e.input_type, e.scale, e.level)


@pytest.mark.parametrize("name", ["sobel", "harris", "polynomial", "feat_hsum", "feat_rot_m1", "feat_rot_m2", "feat_rot_0", "feat_mixed"])
def test_structure(name):
    _, prog, params, sig = load(name)
    for k in ks_for(prog, params):
        check_structure(prog, params, sig, *pack_program(prog, params, sig, k), k)
    if name == "sobel":   # the steps scale: 1 -> 2, 64 -> 128, 130 -> 260 (0 stays 0)
        packed, pparams, _ = pack_program(prog, params, sig, 2)
        assert pparams.rotations == {2 * s for s in params.rotations}
    if name == "feat_rot_m1":   # a step of -1 at vec_size 8 is (-1 mod 8) * k = 7k
        packed, pparams, _ = pack_program(prog, params, sig, 4)
        rots = sorted((int(t.op), t.attributes["RotationAttribute"]) for t in packed.terms() if "RotationAttribute" in t.attributes)
        assert rots == [(int(Op.RotateLeftConst), 28), (int(Op.RotateRightConst), 28)]
        assert pparams.rotations == {28, -28}


def test_inputs_left_untouched_and_k1_copies():
    d, prog, params, sig = load("sobel")
    before = [(t.op, dict(t.attributes)) for t in prog.terms()]
    packed, pparams, psig = pack_program(prog, params, sig, 2)
    assert [(t.op, dict(t.attributes)) for t in prog.terms()] == before
    assert prog.vec_size == sig.vec_size == d["vec_size"] and params.rotations == set(d["rotations"])
    _, prog, params, sig = load("feat_rot_m1")
    same, sp, ss = pack_program(prog, params, sig, 1)
    assert same is not prog and same.name == prog.name and same.vec_size == prog.vec_size
    assert [(t.op, dict(t.attributes)) for t in same.terms()] == [(t.op, dict(t.attributes)) for t in prog.terms()]
    assert (list(sp.prime_bits), sp.rotations, sp.poly_modulus_degree) == (list(params.prime_bits), params.rotations, params.poly_modulus_degree)
    assert ss.vec_size == sig.vec_size and set(ss.inputs) == set(sig.inputs)


@pytest.mark.parametrize("name", ["sobel", "feat_mixed", "polynomial"])
def test_save_load_round_trip(name):
    _, prog, params, sig = load(name)
    k = max_k(prog, params)
    packed, pparams, psig = pack_program(prog, params, sig, k)
    p2, pp2, ps2 = ser.loads(ser.dumps(packed)), ser.loads(ser.dumps(pparams)), ser.loads(ser.dumps(psig))
    assert (p2.name, p2.vec_size) == (packed.name, packed.vec_size)
    assert [(t.op, dict(t.attributes)) for t in p2.terms()] == [(t.op, dict(t.attributes)) for t in packed.terms()]
    assert set(p2.inputs) == set(packed.inputs) and set(p2.outputs) == set(packed.outputs)
    assert (list(pp2.prime_bits), pp2.rotations, pp2.poly_modulus_degree) == (list(pparams.prime_bits), pparams.rotations, pparams.poly_modulus_degree)
    assert ps2.vec_size == psig.vec_size
    assert {n: (e.input_type, e.scale, e.level) for n, e in ps2.inputs.items()} == {n: (e.input_type, e.scale, e.level) for n, e in psig.inputs.items()}
    check_semantics(prog, sig, p2, ps2, k, seed=3)


def plan_shape(prog, N, nprimes, opts, galois=None):
    p = _plan(prog, N, nprimes, opts, 1, galois)
    return p, [(kind, stream, waits, record) for kind, _, stream, waits, record in p["steps"]]


def same_cost(p, q, k):
    """the same plan statistics and ciphertext arena (stride, regions, value offsets).  arena_bytes also counts the staging words of
    the constants encoded on the device, vec_size doubles per Encode (Plan::arenaBytes, rawStride): that part grows k-fold"""
    sp, sq = dict(p["stats"]), dict(q["stats"])
    ap, aq = sp.pop("arena_bytes"), sq.pop("arena_bytes")
    assert sp.pop("arena_bytes_unpacked") == ap and sq.pop("arena_bytes_unpacked") == aq
    assert sq == sp
    assert q["stride"] == p["stride"] and q["regions"] == p["regions"]
    assert sorted(q["values"].values()) == sorted(p["values"].values())
    raw_p, raw_q = ap // 8 - 16 - p["stride"], aq // 8 - 16 - q["stride"]
    assert raw_q == k * raw_p


@pytest.mark.parametrize("opts", [{}, dict(rotation_sums=False), dict(hoist_rotations=False), dict(fuse_sums=False)], ids=["default", "no_rotation_sums", "no_hoist", "no_fuse_sums"])
@pytest.mark.parametrize("name", ["sobel", "harris", "polynomial", "feat_hsum", "feat_mixed"])
def test_plan_cost_unchanged(name, opts):
    """the same steps (kind, stream, events), launches, key switches, rotation-sum calls and ciphertext arena, packed or not"""
    d, prog, params, sig = load(name)
    N, nprimes = params.poly_modulus_degree, len(params.prime_bits)
    k = max_k(prog, params)
    packed, pparams, _ = pack_program(prog, params, sig, k)
    p, shape = plan_shape(prog, N, nprimes, opts)
    q, pshape = plan_shape(packed, N, nprimes, opts)
    assert pshape == shape
    same_cost(p, q, k)
    check_plan(q, packed)


@pytest.mark.parametrize("name", ["sobel", "harris", "feat_hsum"])
def test_power_of_two_keys_scale(name):
    """NAF(r k) is NAF(r) shifted by log2 k: the packed program's power-of-two key steps are the original ones times k, and a plan
    over those keys composes every rotation from as many hops as before"""
    _, prog, params, sig = load(name)
    N, nprimes = params.poly_modulus_degree, len(params.prime_bits)
    k = max_k(prog, params)
    packed, pparams, _ = pack_program(prog, params, sig, k)
    steps = _rotation_key_steps(params, "power_of_two")
    psteps = _rotation_key_steps(pparams, "power_of_two")
    assert sorted(psteps) == sorted(s * k for s in steps)
    p, shape = plan_shape(prog, N, nprimes, {}, {_elt(N, s) for s in steps})
    q, pshape = plan_shape(packed, N, nprimes, {}, {_elt(N, s) for s in psteps})
    assert pshape == shape
    same_cost(p, q, k)
    assert sorted(len(h) for h in q["chains"].values()) == sorted(len(h) for h in p["chains"].values())


def test_errors():
    _, prog, params, sig = load("sobel")
    with pytest.raises(ValueError, match=r"k = 3 is not a power of two"):
        pack_program(prog, params, sig, 3)
    with pytest.raises(ValueError, match=r"k = 0 is not a power of two"):
        pack_program(prog, params, sig, 0)
    with pytest.raises(ValueError, match=r"k = 4 instances of vec_size 4096 need 16384 slots, more than the 8192 of N = 16384"):
        pack_program(prog, params, sig, 4)
    _, p8, pa8, s8 = load("sobel8192")
    with pytest.raises(ValueError, match=r"k = 2 instances of vec_size 8192 need 16384 slots, more than the 8192 of N = 16384"):
        pack_program(p8, pa8, s8, 2)
    _, pp, ppa, pps = load("polynomial")
    with pytest.raises(ValueError, match=r"signature's vec_size 1024 differs from the program's vec_size 4096"):
        pack_program(prog, params, pps, 2)
    vals = valuations(sig, 2, 5)
    with pytest.raises(ValueError, match=r"3 valuations given for k = 2"):
        pack_inputs(vals + vals[:1], sig, 2)
    with pytest.raises(ValueError, match=r"1 valuations given for k = 2"):
        pack_inputs(vals[:1], sig, 2)
    (name,) = sig.inputs
    bad = [vals[0], {"other": vals[1][name]}]
    with pytest.raises(ValueError, match=r"valuation 1 has inputs \['other'\], the signature has \['%s'\]" % name):
        pack_inputs(bad, sig, 2)
    bad = [vals[0], {name: vals[1][name], "extra": vals[1][name]}]
    with pytest.raises(ValueError, match=r"valuation 1 has inputs"):
        pack_inputs(bad, sig, 2)
    bad = [vals[0], {name: np.zeros(3000)}]
    with pytest.raises(ValueError, match=r"input %s of valuation 1 has 3000 values, which does not divide vec_size 4096" % name):
        pack_inputs(bad, sig, 2)
    with pytest.raises(ValueError, match=r"output y has 5 values, not a multiple of k = 2"):
        unpack_outputs({"y": [0.0] * 5}, 2)
