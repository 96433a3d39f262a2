"""Rotations composed from power-of-two Galois keys, without a GPU.  SEAL 3.6's rule is restated here (util::naf and
Evaluator::rotate_internal, as rotate_vector runs it) and checked against the planner's lowering (planner.hpp composeRotations):
the steps every rotation applies, the prefixes chains share, the key switches a plan issues, and the planner invariants of
test_planner.py on every fixture program when only the power-of-two keys are present."""
import re

import pytest

from eva_b200 import Type, program_io as gl
from eva_b200._eva_b200 import Program, _plan, _rotation_key_steps
from oracle import oracle as o

import test_planner as tp


def naf(value):
    """SEAL 3.6 util::naf: `value` as signed powers of two, no two adjacent, lowest first"""
    res, neg, v, i = [], value < 0, abs(value), 0
    while v:
        z = 2 - (v & 3) if v & 1 else 0
        v = (v - z) >> 1
        if z:
            res.append((-z if neg else z) << i)
        i += 1
    return res


def seal_hops(N, steps, elements):
    """Evaluator::rotate_internal: the steps whose key switch rotate_vector(steps) applies, in order, given the Galois elements
    that have keys (a missing key raises KeyError)"""
    if o.galois_elt_from_step(N, steps) in elements:
        return [steps]
    terms = naf(steps)
    if len(terms) == 1:
        raise KeyError(steps)
    out = []
    for t in terms:
        if abs(t) != N // 2:            # no rotation of the N/2 slots
            out += seal_hops(N, t, elements)
    return out


def power_of_two_steps(N, steps):
    """the keys of rotation_keys="power_of_two": the distinct NAF terms of the nonzero steps but +-N/2, ascending"""
    return sorted({t for s in steps if s for t in naf(s) if abs(t) != N // 2})


def elements(N, steps):
    return {o.galois_elt_from_step(N, s) for s in steps}


def rotation_program(N, steps, vec=None):
    """one ciphertext input x and a rotation of x by every SEAL step in `steps` (left for s > 0, right for s < 0), each an output"""
    p = Program("rotations", vec or N // 2)
    x = p._make_input("x", Type.Cipher)
    x._set_attributes({"EncodeAtScaleAttribute": 30, "EncodeAtLevelAttribute": 0})
    terms = {}
    for s in steps:
        r = p._make_left_rotation(x, s) if s > 0 else p._make_right_rotation(x, -s)
        p._make_output("r%d" % s, r)
        terms[s] = r.index
    return p, x.index, terms


def value_steps(p, index, x):
    """the steps whose rotations, applied to x in turn, give the value of term `index` in plan p"""
    step = {t: s for t, _, s in p["rotations"]}
    src = {t: s for t, s, _ in p["rotations"]}
    out = []
    while index != x:
        out.append(step[index])
        index = src[index]
    return out[::-1]


def check_no_rotation_twice(p, N):
    seen = [(s, o.galois_elt_from_step(N, st)) for _, s, st in p["rotations"]]
    assert len(seen) == len(set(seen)), "a rotation is computed twice"


# ---------------------------------------------------------------------------------------------------------------------------

def test_naf_restatement():
    assert naf(0) == [] and naf(1) == [1] and naf(3) == [-1, 4] and naf(-3) == [1, -4] and naf(11) == [-1, -4, 16]
    for v in range(-5000, 5000):
        t = naf(v)
        assert sum(t) == v and all(abs(a) & (abs(a) - 1) == 0 for a in t)
        assert all(abs(b) >= 4 * abs(a) for a, b in zip(t, t[1:]))   # non-adjacent, lowest first


@pytest.mark.parametrize("N", [1024, 2048])
def test_every_step_lowered_as_seal(N):
    """every step 0 < |s| < N/2 under the power-of-two keys: the steps of each rotation's chain are SEAL's, the value the plan
    computes is that chain, and the plan's hops are exactly the chain prefixes that no program rotation computes, each once"""
    steps = [s for s in range(-(N // 2) + 1, N // 2) if s]
    keys = power_of_two_steps(N, steps)
    assert keys == sorted(t for j in range(N.bit_length()) for t in (-(1 << j), 1 << j) if (1 << j) < N // 2)
    elts = elements(N, keys)
    prog, x, terms = rotation_program(N, steps)

    def elts_of(chain):
        return tuple(o.galois_elt_from_step(N, a) for a in chain)
    for opts in ({}, dict(rotation_chunk=1), dict(hoist_mod_up=False)):
        p = _plan(prog, N, 3, opts, 1, elts)
        composed = 0
        for s, t in terms.items():
            want = seal_hops(N, s, elts)
            assert p["chains"][t] == want, s
            assert elts_of(value_steps(p, t, x)) == elts_of(want), s
            composed += len(want) > 1
        assert p["stats"]["composed_rotations"] == composed > 0
        # the hops are the proper prefixes of the chains that no program rotation computes, each once
        program_chains = {elts_of(c) for c in p["chains"].values()}
        prefixes = {elts_of(c[:j]) for c in p["chains"].values() for j in range(1, len(c))}
        hops = [t for t, _, _ in p["rotations"] if t not in p["chains"]]
        hop_chains = [elts_of(value_steps(p, t, x)) for t in hops]
        assert sorted(hop_chains) == sorted(prefixes - program_chains)
        assert len(hops) == p["stats"]["composed_hops"] and len(p["rotations"]) == len(terms) + len(hops)


def test_prefix_with_a_direct_key_of_its_sum_is_not_shared():
    """keys {-1, -4, 16, -5}: rot_-5(x) uses the -5 key; naf(11) = [-1, -4, 16] goes through rot_-1(x) (the program's rotation: a
    single-term prefix) and a hop rot_-4(rot_-1(x)), never through rot_-5(x)"""
    N = 1024
    prog, x, terms = rotation_program(N, [-5, -1, 11])
    elts = elements(N, [-1, -4, 16, -5])
    p = _plan(prog, N, 3, {}, 1, elts)
    assert p["chains"] == {terms[-5]: [-5], terms[-1]: [-1], terms[11]: [-1, -4, 16]}
    hop = p["sources"][terms[11]]
    assert hop >= prog.terms()[-1].index + 1 and hop != terms[-5]
    assert p["sources"][hop] == terms[-1] and terms[-5] not in p["sources"]
    assert sorted((s, st) for t, s, st in p["rotations"] if t == hop) == [(terms[-1], -4)]
    assert len(p["rotations"]) == 4 and p["stats"]["composed_rotations"] == 1 and p["stats"]["composed_hops"] == 1


def test_keyless_rotation_is_a_prefix_of_a_longer_chain():
    """keys {1, 4, 16}: rot_5(x) is the chain [1, 4]; rot_21(x) = [1, 4, 16] continues from rot_5(x) itself"""
    N = 1024
    prog, x, terms = rotation_program(N, [21, 5])
    p = _plan(prog, N, 3, {}, 1, elements(N, [1, 4, 16]))
    assert p["chains"] == {terms[5]: [1, 4], terms[21]: [1, 4, 16]}
    assert p["sources"][terms[21]] == terms[5]
    assert p["sources"][p["sources"][terms[5]]] == x
    assert len(p["rotations"]) == 3 and p["stats"]["composed_hops"] == 1


def test_half_ring_term_is_dropped():
    """a step s and s - N/2 share their element: N/2 - 1 (naf [-1, N/2]) uses the key of -1 and 3N/8 (naf [-N/8, N/2]) that of
    -N/8 directly; N/2 - 3 (naf [1, -4, N/2]) without the key of -3 is the chain [1, -4]"""
    N = 1024
    prog, x, terms = rotation_program(N, [N // 2 - 1, 3 * N // 8, N // 2 - 3, 3])
    elts = elements(N, [-1, 1, -4, 4, -N // 8])
    p = _plan(prog, N, 3, {}, 1, elts)
    assert naf(N // 2 - 3) == [1, -4, N // 2] and naf(3 * N // 8) == [-N // 8, N // 2]
    assert p["chains"][terms[N // 2 - 1]] == [N // 2 - 1] == seal_hops(N, N // 2 - 1, elts)
    assert p["chains"][terms[3 * N // 8]] == [3 * N // 8] == seal_hops(N, 3 * N // 8, elts)
    assert p["chains"][terms[N // 2 - 3]] == [1, -4] == seal_hops(N, N // 2 - 3, elts)
    assert p["chains"][terms[3]] == [-1, 4]
    check_no_rotation_twice(p, N)


def test_missing_hop_key_names_step_term_and_element():
    N = 1024
    prog, _, _ = rotation_program(N, [3])
    e = o.galois_elt_from_step(N, -1)
    with pytest.raises(ValueError, match=r"Galois key not present.*rotation by 3 steps.*term -1 \(Galois element %d\)" % e):
        _plan(prog, N, 3, {}, 1, elements(N, [1, 4]))
    with pytest.raises(ValueError, match=r"rotation by 5 steps.*term 4 \(Galois element %d\)" % o.galois_elt_from_step(N, 4)):
        _plan(rotation_program(N, [5])[0], N, 3, {}, 1, elements(N, [1]))   # naf(5) = [1, 4]
    with pytest.raises(ValueError):
        _plan(rotation_program(N, [8])[0], N, 3, {}, 1, elements(N, [1, 2, 4]))   # a power of two without its key


def test_key_steps():
    params = gl.build_program(gl.load_json("sobel"))[1]
    N = params.poly_modulus_degree
    assert _rotation_key_steps(params, "program") == sorted(params.rotations)
    assert _rotation_key_steps(params, "power_of_two") == power_of_two_steps(N, params.rotations) == [1, 2, 64, 128]
    wide = gl.build_program(gl.load_json("wide4096"))[1]
    assert _rotation_key_steps(wide, "power_of_two") == power_of_two_steps(wide.poly_modulus_degree, wide.rotations) == \
        [-16, -8, -4, -2, -1, 1, 2, 4, 8, 16, 32, 64]
    with pytest.raises(ValueError, match="rotation_keys"):
        _rotation_key_steps(params, "powers")


# ---------------------------------------------------------------------------------------------------------------------------
# the workloads and the fixture programs

WORKLOADS = {"sobel": (8, 8), "harris": (32, 32), "wide64": (None, 84), "wide4096": (126, 168)}


def program_keys(name, rotation_keys):
    d = gl.load_json(name)
    N = d["poly_modulus_degree"]
    steps = _rotation_key_steps(gl.build_program(d)[1], rotation_keys)
    return elements(N, steps)


@pytest.mark.parametrize("name", sorted(WORKLOADS))
def test_workload_key_switches(name):
    """key switches per instance -- the program's distinct rotations plus the plan's hops -- with the program's keys and with the
    power-of-two keys; the plan issues no rotation twice (it may issue fewer: rotations whose every use has weight 0 are elided)"""
    now, composed = WORKLOADS[name]
    prog, N, k = tp.program(name)
    full = _plan(prog, N, k, {}, 1)
    if now is not None:
        assert len(full["chains"]) + full["stats"]["composed_hops"] == now
    p = _plan(prog, N, k, {}, 1, program_keys(name, "power_of_two"))
    assert len(p["chains"]) + p["stats"]["composed_hops"] == composed
    assert len(p["rotations"]) <= composed
    check_no_rotation_twice(p, N)
    elts = program_keys(name, "power_of_two")
    assert p["chains"].keys() == full["chains"].keys()
    for t, chain in p["chains"].items():
        assert full["chains"][t] == [full["chains"][t][0]] and chain == seal_hops(N, full["chains"][t][0], elts)


def test_sobel_plan_shape():
    """Sobel under {1, 2, 64, 128}: no plan-owned hop; a hoist group on x (1, 2, 64, 128) and groups on rot1(x) and rot2(x) (64, 128)"""
    prog, N, k = tp.program("sobel")
    p = _plan(prog, N, k, {}, 1, program_keys("sobel", "power_of_two"))
    st = p["stats"]
    assert st["composed_rotations"] == 4 and st["composed_hops"] == 0 and st["hoist_groups"] == 3
    by_src = {}
    for t, s, step in p["rotations"]:
        by_src.setdefault(s, []).append(step)
    # rot_65(x) = rot_64(rot_1(x)) has weight 0 in both sums: elided, as it is with the program's keys
    rot1, rot2 = [t for t, _, step in p["rotations"] if step in (1, 2)]
    assert sorted(by_src[rot1]) == [128] and sorted(by_src[rot2]) == [64, 128] and len(by_src) == 3
    assert len(p["rotations"]) == len(_plan(prog, N, k, {}, 1)["rotations"]) == 7


@pytest.mark.parametrize("name", tp.PROGRAMS + ["wide4096"])
def test_program_keys_plan_unchanged(name):
    """with every key of the program present, the plan is the plan built without an element set"""
    prog, N, k = tp.program(name)
    for opts in ({}, dict(rotation_sums=False)):
        assert _plan(prog, N, k, opts, 1, program_keys(name, "program")) == _plan(prog, N, k, opts, 1)


class _Node:
    def __init__(self, index):
        self.index, self.operands = index, []


class PlanOperands:
    """the program's terms and the plan's hops, with the operands the plan reads: a hop or a composed rotation reads the term that
    `sources` names (test_planner's check_operands then checks the plan's reads)"""

    def __init__(self, prog, sources):
        real = {t.index: t for t in prog.terms()}
        self.nodes = {i: _Node(i) for i in list(real) + list(sources)}
        for i, n in self.nodes.items():
            n.operands = [self.nodes[sources[i]]] if i in sources else [self.nodes[x.index] for x in real[i].operands]

    def terms(self):
        return list(self.nodes.values())


@pytest.mark.parametrize("option", sorted(tp.OPTIONS))
@pytest.mark.parametrize("name", tp.PROGRAMS)
def test_plan_invariants_power_of_two(name, option):
    """test_planner's invariants with the power-of-two keys: one-offset-per-value and packed, deterministic"""
    opts, batch = tp.OPTIONS[option]
    prog, N, k = tp.program(name)
    elts = program_keys(name, "power_of_two")

    def plan(limit=0):
        return _plan(prog, N, k, dict(opts, arena_limit=limit), batch, elts)
    p = plan()
    tp.check_plan(p, PlanOperands(prog, p["sources"]))
    assert plan() == p
    assert p["stats"]["packed"] == 0
    limit = p["stats"]["arena_bytes_unpacked"] - 1
    try:
        q = plan(limit)
    except RuntimeError as e:
        m = re.search(r"needs (\d+) bytes packed \((\d+) bytes unpacked\)", str(e))
        assert m and int(m.group(1)) == int(m.group(2)) == limit + 1, e
        return
    assert q["stats"]["packed"] == 1 and q["stats"]["arena_bytes"] <= limit
    tp.check_plan(q, PlanOperands(prog, q["sources"]))
    assert plan(limit) == q
