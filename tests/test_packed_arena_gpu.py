"""Packed plan arenas on the GPU: with an arena_limit below what the one-offset-per-value layout takes, the plan reuses
the storage of dead values (eva_b200/csrc/host/arena_packer.hpp).  Its outputs are the unpacked plan's, bit for bit,
in every scheduler mode; a program whose unpacked arena exceeds the card's memory runs in a few GB; plans that fit
are laid out as before."""
import re
import time

import numpy as np
import pytest

from eva_b200 import program_io as gl
from oracle import oracle as o
from oracle_exec import OracleProgram

pytestmark = pytest.mark.gpu

FEATURES = ["feat_bin_mul_11", "feat_bin_sub_01", "feat_unary", "feat_rot_m1", "feat_rot_0", "feat_mixed",
            "feat_transparent", "feat_hsum", "feat_deep"]


def context(d, seed=1):
    from eva_b200 import b200
    N = d["poly_modulus_degree"]
    orc = o.Oracle(N, d["prime_bits"]).keygen(seed)
    op = OracleProgram(d, orc)
    op.prepare_keys()
    pub = b200.context_from_raw_keys(N, orc.primes, op.rk, {int(e): k for e, k in op.gks.items()})
    return orc, op, pub


def valuation(d, orc, rng, lo=0.0, hi=0.2, seed=11):
    from eva_b200 import b200
    val, inputs_o = b200.B200Valuation(), {}
    for name, info in d["signature"].items():
        x = rng.uniform(lo, hi, d["vec_size"])
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


def assert_same(a, b):
    assert sorted(a.names()) == sorted(b.names())
    for n in a.names():
        ka, xa, sa = a.get(n)
        kb, xb, sb = b.get(n)
        assert ka == kb and sa == sb
        assert np.array_equal(np.asarray(xa), np.asarray(xb)), n


def packed_vs_unpacked(d, n_vals=1, **opts):
    """the same valuations through the default layout and through a packed one (limit = unpacked bytes - 1)"""
    prog, _, _, _ = gl.build_program(d)
    orc, _, pub = context(d)
    rng = np.random.default_rng(2)
    vals = [valuation(d, orc, rng, seed=11 + i)[0] for i in range(n_vals)]
    F = min(opts.get("fuse", 1), n_vals)
    replicas = range((n_vals + F - 1) // F)
    pub.set_options(**opts)
    want = pub.execute_batch(prog, vals)
    st = pub.plan_stats(prog, F, 0)
    assert st["packed"] == 0 and st["arena_bytes"] == st["arena_bytes_unpacked"] and st["reuse_waits"] == 0
    limit = st["arena_bytes_unpacked"] - 1
    pub.set_options(**opts, arena_limit=limit)
    for _ in range(2):   # the second call replays the captured graph
        got = pub.execute_batch(prog, vals)
        for a, b in zip(got, want):
            assert_same(a, b)
    stats = [pub.plan_stats(prog, F, r) for r in replicas]
    for s in stats:
        assert s["packed"] == 1 and s["arena_bytes"] <= limit and s["arena_bytes_unpacked"] == limit + 1
    return stats[0]


@pytest.mark.parametrize("name", ["sobel", "harris", "wide64", "polynomial"])
def test_packed_outputs_equal_unpacked(name):
    packed_vs_unpacked(gl.load_json(name))


@pytest.mark.parametrize("name", FEATURES)
def test_packed_feature_programs(name):
    """a program with no storage to reuse (every value is an input, an output, or read by the step that writes the only
    other value) packs to its unpacked size: a limit below that is refused with both byte counts"""
    try:
        packed_vs_unpacked(gl.load_json(name))
    except RuntimeError as e:
        m = re.search(r"needs (\d+) bytes packed \((\d+) bytes unpacked\), more than the limit of (\d+)", str(e))
        assert m and m.group(1) == m.group(2) and int(m.group(3)) == int(m.group(1)) - 1, e


@pytest.mark.parametrize("graph,streams", [(False, 1), (False, 8), (True, 1), (True, 8)])
@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_packed_scheduler_modes(name, graph, streams):
    packed_vs_unpacked(gl.load_json(name), use_graph=graph, num_streams=streams)


@pytest.mark.parametrize("chunk", [1, 16])
@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_packed_rotation_chunks(name, chunk):
    packed_vs_unpacked(gl.load_json(name), rotation_chunk=chunk)


@pytest.mark.parametrize("fuse", [1, 2])
def test_packed_batched_plans(fuse):
    st = packed_vs_unpacked(gl.load_json("sobel"), n_vals=4, fuse=fuse)
    assert st["arena_bytes"] < st["arena_bytes_unpacked"]


@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_packed_approx_hoist(name):
    st = packed_vs_unpacked(gl.load_json(name), approx_hoist=True)
    assert st["lazy_calls"] > 0


def test_packed_without_constant_cache_and_fused_sums():
    packed_vs_unpacked(gl.load_json("sobel"), cache_constants=False, fuse_sums=False)


def test_packed_zero_digit_falls_back_to_the_exact_path():
    """as test_executor_parity.test_zero_digit_falls_back_to_the_exact_path, with both the shared-mod-up plan and the
    plan it is rebuilt without packed"""
    from eva_b200 import b200
    d = gl.load_json("sobel")
    prog, _, _, _ = gl.build_program(d)
    orc, op, pub = context(d)
    unpacked = []
    for hoist in (True, False):
        pub.set_options(hoist_mod_up=hoist)
        unpacked.append(pub.plan_stats(prog)["arena_bytes_unpacked"])
    limit = min(unpacked) - 1
    pub.set_options(arena_limit=limit)
    rng = np.random.default_rng(4)
    (name_, info), = d["signature"].items()
    ell = orc.k - 1 - info["level"]
    ct = orc.encrypt(orc.encode(rng.uniform(0, 1, d["vec_size"]), 2.0 ** info["scale"], ell), seed=3)
    c1 = np.stack([orc.ntt_inv(ct[1, i], i) for i in range(ell)])
    c1[1, 7] = 0                                     # one zero coefficient in digit 1
    ct[1] = np.stack([orc.ntt_fwd(c1[i], i) for i in range(ell)])
    val = b200.B200Valuation()
    val.set_cipher(name_, ct, 2.0 ** info["scale"])
    V = op.run({name_: ("cipher", ct, 2.0 ** info["scale"])})
    assert pub.plan_stats(prog)["packed"] == 1
    for _ in range(2):                               # first call falls back, second runs on the rebuilt plan
        out = pub.execute(prog, val)
        for oname, oid in d["outputs"].items():
            assert np.array_equal(out.get(oname)[1], V[oid][1])
    st = pub.plan_stats(prog)                        # the plan without the shared mod-up, packed too
    assert st["packed"] == 1 and st["arena_bytes"] <= limit and st["arena_bytes_unpacked"] == unpacked[1]


def test_plans_that_fit_keep_the_existing_layout():
    for name in ("sobel", "harris"):
        d = gl.load_json(name)
        prog, _, _, _ = gl.build_program(d)
        _, _, pub = context(d)
        st = pub.plan_stats(prog)
        assert st["packed"] == 0 and st["reuse_waits"] == 0
        assert st["arena_bytes"] == st["arena_bytes_unpacked"] > 0
        assert st["constant_bytes"] > 0


def test_limit_below_the_packed_peak_raises_and_overwritten_values_are_not_read_back():
    d = gl.load_json("sobel")
    prog, _, _, terms = gl.build_program(d)
    orc, op, pub = context(d)
    rng = np.random.default_rng(6)
    val, inputs_o = valuation(d, orc, rng)
    unpacked = pub.plan_stats(prog)["arena_bytes_unpacked"]
    pub.set_options(arena_limit=unpacked - 1)
    out = pub.execute(prog, val)
    V = op.run(inputs_o)
    for oname, oid in d["outputs"].items():
        assert np.array_equal(out.get(oname)[1], V[oid][1])
    # inputs and outputs are kept; an intermediate's storage has been reused and cannot be read back
    for tid in list(d["inputs"].values()) + list(d["outputs"].values()):
        arr, scale = pub.debug_value(prog, terms[tid].index)
        assert np.array_equal(arr, V[tid][1]) and scale == V[tid][2]
    kept = {a for t in d["terms"] if t["op"] == "Output" for a in t["args"]}
    inner = [t["id"] for t in d["terms"] if t["op"] in ("Relinearize", "Rescale") and t["id"] not in kept]
    assert inner
    for tid in inner:
        with pytest.raises(RuntimeError, match="packed arena"):
            pub.debug_value(prog, terms[tid].index)
    peak = pub.plan_stats(prog)["arena_bytes"]
    pub.set_options(arena_limit=peak - 1)
    with pytest.raises(RuntimeError) as e:
        pub.execute(prog, val)
    assert str(peak) in str(e.value) and str(peak - 1) in str(e.value) and str(unpacked) in str(e.value)


# ---- a program whose one-offset-per-value arena does not fit on the card

def chains_program(n_chains, depth, vec=8192):
    """n_chains interleaved chains v <- (v << a) + v - (v >> (vec - a)), summed at the end; the sum and its 8th power are
    the outputs (the three squarings make the modulus chain long enough for N = 16384).  With vec = N/2 the two rotations
    are the same permutation of every slot, so each step keeps the chain's value and adds only the noise of two key
    switches (with fewer slots than N/2 they differ on the noise, which would grow threefold per step)."""
    from eva import EvaProgram, Input, Output
    p = EvaProgram("chains_%dx%d" % (n_chains, depth), vec_size=vec)
    with p:
        x = Input("x")
        vs = [x << (c + 1) for c in range(n_chains)]
        for k in range(depth):
            a = 1 + k % 7
            vs = [(v << a) + v - (v >> (vec - a)) for v in vs]
        s = vs[0]
        for v in vs[1:]:
            s = s + v
        Output("s", s)
        for _ in range(3):
            s = s * s
        Output("y", s)
    p.set_output_ranges(20)
    p.set_input_scales(30)
    return p


def program_dict(prog, params, sig):
    """a compiled Program in the JSON form program_io / oracle_exec read"""
    d = {"name": prog.name, "vec_size": prog.vec_size, "poly_modulus_degree": params.poly_modulus_degree,
         "prime_bits": list(params.prime_bits), "rotations": sorted(params.rotations),
         "signature": {n: {"type": i.input_type.name, "scale": i.scale, "level": i.level} for n, i in sig.inputs.items()},
         "inputs": {n: t.index for n, t in prog.inputs.items()}, "outputs": {n: t.index for n, t in prog.outputs.items()}, "terms": []}
    keys = {"RotationAttribute": "rotation", "EncodeAtScaleAttribute": "scale", "EncodeAtLevelAttribute": "level",
            "RescaleDivisorAttribute": "divisor", "RangeAttribute": "range"}
    for t in prog.terms():
        a = t.attributes
        e = {"id": t.index, "op": t.op.name, "args": [x.index for x in t.operands]}
        e.update({keys[k]: v for k, v in a.items() if k in keys})
        if "TypeAttribute" in a:
            e["type"] = a["TypeAttribute"].name
        if "ConstantValueAttribute" in a:
            e["const"] = list(a["ConstantValueAttribute"])
        d["terms"].append(e)
    return d


def test_small_chains_program_packed_is_bit_identical_to_the_oracle():
    from eva.ckks import CKKSCompiler
    compiled, params, sig = CKKSCompiler().compile(chains_program(4, 3))
    assert params.poly_modulus_degree >= 16384
    d = program_dict(compiled, params, sig)
    prog, _, _, _ = gl.build_program(d)
    orc, op, pub = context(d)
    val, inputs_o = valuation(d, orc, np.random.default_rng(8), lo=0.0, hi=1.0 / 32)
    V = op.run(inputs_o)
    unpacked = pub.plan_stats(prog)["arena_bytes_unpacked"]
    for limit in (0, unpacked - 1):
        pub.set_options(arena_limit=limit)
        out = pub.execute(prog, val)
        assert pub.plan_stats(prog)["packed"] == (1 if limit else 0)
        for oname, oid in d["outputs"].items():
            kind, arr, scale = out.get(oname)
            assert np.array_equal(arr, V[oid][1]) and scale == V[oid][2]


def test_program_larger_than_device_memory_runs_packed():
    import torch
    from eva import evaluate
    from eva.ckks import CKKSCompiler
    from eva.metric import valuation_mse
    from eva.seal import generate_keys
    prog = chains_program(64, 200)
    compiled, params, sig = CKKSCompiler().compile(prog)
    assert params.poly_modulus_degree >= 16384
    limit = 4 << 30
    pub, sec = generate_keys(params)
    pub.set_options(use_graph=False, arena_limit=limit)   # set before the plan exists: the unpacked arena is never allocated
    t0 = time.perf_counter()
    st = pub.plan_stats(compiled)
    t_plan = time.perf_counter() - t0
    _, total = torch.cuda.mem_get_info()
    assert st["arena_bytes_unpacked"] > total, (st["arena_bytes_unpacked"], total)
    assert st["packed"] == 1 and st["arena_bytes"] <= limit
    rng = np.random.default_rng(3)
    inputs = {"x": list(rng.uniform(0, 1.0 / 32, 8192))}
    enc = pub.encrypt(inputs, sig)
    pub.execute(compiled, enc)                              # warm-up
    t0 = time.perf_counter()
    out = pub.execute(compiled, enc)
    t_run = time.perf_counter() - t0
    assert valuation_mse(sec.decrypt(out, sig), evaluate(prog, inputs)) < 0.01
    print("\nchains 64x200: %d terms, N=%d, unpacked %.1f GB, packed %.2f GB, %d reuse waits, plan %.2f s, execute %.3f s"
          % (len(compiled.terms()), params.poly_modulus_degree, st["arena_bytes_unpacked"] / 1e9, st["arena_bytes"] / 1e9,
             st["reuse_waits"], t_plan, t_run))
