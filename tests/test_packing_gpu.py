"""Slot packing on the GPU.  A packed program is an ordinary program, so it runs on the existing kernels unchanged:
- a packed Sobel / polynomial built by an independent restatement of the packing rule (on the workload dumps) equals pack_program's
  output term by term, and every intermediate ciphertext of its execution is bit-identical to the oracle's;
- packed Sobel, Harris and polynomial with distinct inputs per instance, encrypted with the public and with the secret (seeded)
  context: every unpacked request meets the MSE criterion against evaluate() of the unpacked program;
- B200Server(pparams, ...) serves packed tenants (two tenants; power-of-two keys; seeded inline keys with a c1 cache; paging), sync
  and async, with outputs bit-identical to each tenant's own packed context."""
import json

import numpy as np
import pytest

from eva_b200 import evaluate, program_io as gl
from eva_b200.ckks import pack_inputs, pack_program, unpack_outputs

import test_executor_parity as tep

pytestmark = pytest.mark.gpu

MSE = 0.01   # the reference's acceptance criterion (tests/common.py), HE against plaintext
WORKLOADS = {"sobel": 2, "harris": 2, "polynomial": 4}
RANGE = {"sobel": (0.0, 0.2), "harris": (0.0, 0.2), "polynomial": (-1.0, 1.0)}


def packed_dict(d, k):
    """the packing rule restated on a program dump: vec_size v*k, rotation steps (r mod v)*k, dense constants interleaved, the
    rotation keys of the scaled ciphertext steps"""
    v = d["vec_size"]
    p = json.loads(json.dumps(d))
    p["name"], p["vec_size"] = "%s.pack%d" % (d["name"], k), v * k
    steps = set()
    for t in p["terms"]:
        if t["op"] in ("RotateLeftConst", "RotateRightConst"):
            t["rotation"] = (t["rotation"] % v) * k
            if t.get("type") != "Raw":
                steps.add(t["rotation"] if t["op"] == "RotateLeftConst" else -t["rotation"])
        if t["op"] == "Constant" and len(t["const"]) > 1:
            t["const"] = [c for c in t["const"] for _ in range(k)]
    p["rotations"] = sorted(steps)
    return p


def same_program(a, b):
    ta, tb = a.terms(), b.terms()
    assert (a.name, a.vec_size, len(ta)) == (b.name, b.vec_size, len(tb))
    pa, pb = {t.index: i for i, t in enumerate(ta)}, {t.index: i for i, t in enumerate(tb)}
    for x, y in zip(ta, tb):
        assert x.op == y.op and dict(x.attributes) == dict(y.attributes)
        assert [pa[o.index] for o in x.operands] == [pb[o.index] for o in y.operands]
    assert {n: pa[t.index] for n, t in a.inputs.items()} == {n: pb[t.index] for n, t in b.inputs.items()}
    assert {n: pa[t.index] for n, t in a.outputs.items()} == {n: pb[t.index] for n, t in b.outputs.items()}


@pytest.mark.parametrize("name,k", [("sobel", 2), ("polynomial", 4)])
def test_packed_bit_exact_against_oracle(name, k, monkeypatch):
    d = gl.load_json(name)
    pd = packed_dict(d, k)
    prog, params, sig, _ = gl.build_program(d)
    packed, pparams, psig = pack_program(prog, params, sig, k)
    same_program(gl.build_program(pd)[0], packed)
    assert pparams.rotations == set(pd["rotations"]) and psig.vec_size == pd["vec_size"]
    load = gl.load_json
    monkeypatch.setattr(gl, "load_json", lambda n: pd if n == pd["name"] else load(n))
    lo, hi = RANGE[name]
    r = tep.run_both(pd["name"], lo=lo, hi=hi)
    assert r[4] >= {"sobel": 61, "polynomial": 14}[name]   # every ciphertext and plaintext term
    r = tep.run_both(pd["name"], lo=lo, hi=hi, fuse_sums=True)
    assert r[4] > 0


def requests(name, sig, k, seed):
    rng = np.random.default_rng(seed)
    lo, hi = RANGE[name]
    return [{n: rng.uniform(lo, hi, sig.vec_size) for n in sig.inputs} for _ in range(k)]


def mse_each(prog, vals, outs):
    worst = 0.0
    for v, o in zip(vals, outs):
        want = evaluate(prog, {n: list(x) for n, x in v.items()})
        for n in want:
            worst = max(worst, float(np.mean((np.asarray(want[n]) - o[n]) ** 2)))
    return worst


@pytest.mark.parametrize("name", sorted(WORKLOADS))
def test_packed_accuracy(name):
    from eva_b200 import b200
    k = WORKLOADS[name]
    d = gl.load_json(name)
    prog, params, sig, _ = gl.build_program(d)
    packed, pparams, psig = pack_program(prog, params, sig, k)
    public_ctx, secret_ctx = b200.generate_keys(pparams, seed=5)
    for i, enc in enumerate((public_ctx.encrypt, secret_ctx.encrypt)):
        vals = requests(name, sig, k, 10 + i)
        assert len({float(v[n][0]) for v in vals for n in v}) == k * len(sig.inputs)   # distinct per instance
        ins = enc(pack_inputs(vals, sig, k), psig)
        outs = unpack_outputs(secret_ctx.decrypt(public_ctx.execute(packed, ins), psig), k)
        assert len(outs) == k and all(len(o[n]) == sig.vec_size for o in outs for n in o)
        worst = mse_each(prog, vals, outs)
        assert worst < MSE, (name, i, worst)


def _same(a, b, names, what):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        for n in names:
            assert np.array_equal(x.get(n)[1], y.get(n)[1]), (what, n)


SERVERS = {
    "two_tenants": (dict(capacity=2), {}, 2),
    "power_of_two": (dict(capacity=2, rotation_keys="power_of_two"), dict(rotation_keys="power_of_two"), 2),
    "seeded_c1": (dict(capacity=2, hoist_constants="inline", key_storage="seeded", c1_cache=1), {}, 2),
    "paged": (dict(capacity=2, max_tenants=3), {}, 3),
}


@pytest.mark.parametrize("variant", sorted(SERVERS))
def test_server_serves_packed_tenants(variant):
    from eva_b200 import b200
    skw, gkw, tenants = SERVERS[variant]
    d = gl.load_json("sobel")
    prog, params, sig, _ = gl.build_program(d)
    packed, pparams, psig = pack_program(prog, params, sig, 2)
    srv = b200.B200Server(pparams, **skw)
    ctxs = [b200.generate_keys(pparams, seed=70 + t, **gkw) for t in range(tenants)]
    for t, (pub, _) in enumerate(ctxs):
        assert srv.add_keys(pub) == t
    for i, order in enumerate(([0, 1, 1, 0], [tenants - 1, 0], [1, tenants - 1])):
        rq, vals = [], []
        for j, t in enumerate(order):
            v = requests("sobel", sig, 2, 100 * i + j)
            vals.append(v)
            pub, sec = ctxs[t]
            rq.append((t, sec.encrypt(pack_inputs(v, sig, 2), psig) if j % 2 else pub.encrypt(pack_inputs(v, sig, 2), psig)))
        outs = srv.execute_batch(packed, rq)
        own = [ctxs[t][0].execute_batch(packed, [val])[0] for t, val in rq]
        _same(outs, own, d["outputs"], (variant, order))
        h = srv.execute_batch_async(packed, rq)
        _same(srv.execute_batch_result(h), own, d["outputs"], (variant, order, "async"))
        for (t, _), o, v in zip(rq, outs, vals):   # and each packed request decrypts to its two instances
            assert mse_each(prog, v, unpack_outputs(ctxs[t][1].decrypt(o, psig), 2)) < MSE
    info = srv.bank_info()
    if variant == "paged":
        assert info["evictions"] > 0
    if variant == "seeded_c1":
        assert info["key_storage"] == "seeded" and info["c1_cache"] == 1
