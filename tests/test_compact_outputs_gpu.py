"""Compact responses on the GPU: the packed words of every execution path equal the Python-integer compaction of the same batch's
full outputs; collect's zero-digit redo stays compact and exact; the client's integers equal an exact decryption with the exported
secret key; decryption stays within 2^-p of the full ciphertext's; and with the option off nothing changes."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from eva_b200 import program_io as gl
from oracle import oracle as o
from oracle_exec import OracleProgram
from test_compact_outputs import compact_ref, fields, pack_ref
from test_seeded_inputs_gpu import _ctx, client_inputs
from test_stored_inputs_gpu import request

pytestmark = pytest.mark.gpu
u64p = C.POINTER(C.c_uint64)
GOLDEN = "image_processing_baboon.npz"

_ORACLES = {}


def oracle_for(N, primes):
    key = (N, tuple(primes))
    if key not in _ORACLES:
        _ORACLES[key] = o.Oracle(N, primes=list(primes))
    return _ORACLES[key]


def expected_compact(m, prog, primes, name, full, p):
    """(words, bits, scale) of the full output `full` = (kind, ct [2][ell][N] NTT form, scale) by the definition, or None (stays full)"""
    kind, ct, scale = full
    if kind != "cipher" or ct.shape[0] != 2:
        return None
    ell, N = ct.shape[1], ct.shape[2]
    rng_bits = prog.outputs[name].attributes["RangeAttribute"]
    compact, shift, bits, cscale = m._compact_shape(list(primes), ell, scale, rng_bits, p, N)
    if not compact:
        return None
    orc = oracle_for(N, primes)
    Q = math.prod(int(q) for q in primes[:ell])
    words = []
    for j in range(2):
        rows = [orc.ntt_inv(ct[j, i], i) for i in range(ell)]
        xs = [int(v) for v in rows[0]] if ell == 1 else crt_rows(rows, primes[:ell])
        words.append(pack_ref(compact_ref(xs, Q, shift, bits), bits))
    return np.stack(words), bits, cscale


def crt_rows(rows, primes):
    Q = math.prod(int(q) for q in primes)
    acc = [0] * len(rows[0])
    for r, q in zip(rows, primes):
        q = int(q)
        mq = Q // q
        f = mq * pow(mq, -1, q)
        for i, v in enumerate(r):
            acc[i] += int(v) * f
    return [x % Q for x in acc]


def check_batch(m, prog, primes, outs_full, outs_compact, p, what):
    assert len(outs_full) == len(outs_compact)
    compacted = 0
    for i, (f, c) in enumerate(zip(outs_full, outs_compact)):
        for name in f.names():
            want = expected_compact(m, prog, primes, name, f.get(name), p)
            got = c.get(name)
            if want is None:
                assert got[0] == f.get(name)[0] and np.array_equal(got[1], f.get(name)[1]), (what, i, name)
                continue
            assert got[0] == "compact_cipher", (what, i, name)
            assert c.compact_bits(name) == want[1] and got[2] == want[2], (what, i, name)
            assert np.array_equal(got[1], want[0]), (what, i, name)
            compacted += 1
    return compacted


def _m():
    from eva_b200 import _eva_b200 as m
    return m


# ------------------------------------------------------------------------------------------------ bit-exact words, B200Public
@pytest.mark.parametrize("name", ["sobel", "harris", "polynomial"])
def test_public_paths_are_bit_exact(name):
    d, prog, params, sig, pub, sec = _ctx(name)
    primes = list(pub.primes())
    B = 3
    encs = [sec.encrypt(client_inputs(d, i), sig) for i in range(B)]
    full = pub.execute_batch(prog, encs)
    pub.set_options(compact_outputs=10)
    got = pub.execute_batch(prog, encs)
    assert check_batch(_m(), prog, primes, full, got, 10, "execute_batch") == B * len(d["outputs"])
    h = pub.execute_batch_async(prog, encs, 3)
    check_batch(_m(), prog, primes, full, pub.execute_batch_result(h), 10, "async")
    pub.set_options(compact_outputs=10, fuse=B)
    check_batch(_m(), prog, primes, full, pub.execute_batch(prog, encs), 10, "one fused chunk")
    pub.set_options()
    again = pub.execute_batch(prog, encs)
    for a, b in zip(full, again):
        for n in a.names():
            assert a.get(n)[0] == "cipher" and np.array_equal(a.get(n)[1], b.get(n)[1])


def test_two_prime_output_is_bit_exact():
    """Sobel at one level more: its output keeps two primes, whose 128 bits per coefficient shrink to b"""
    from eva_b200 import b200
    d = gl.load_json("sobel")
    d = dict(d, prime_bits=[60] + list(d["prime_bits"]))
    prog, params, sig, _ = gl.build_program(d)
    pub, sec = b200.generate_keys(params, seed=8)
    encs = [sec.encrypt(client_inputs(d, i), sig) for i in range(2)]
    full = pub.execute_batch(prog, encs)
    assert full[0].get(list(d["outputs"])[0])[1].shape[1] == 2
    pub.set_options(compact_outputs=12)
    assert check_batch(_m(), prog, list(pub.primes()), full, pub.execute_batch(prog, encs), 12, "two primes") == 2


def test_other_outputs_stay_as_they_are():
    """a size-3 output ciphertext stays full; the size-2 ciphertext next to it is compacted (the non-ciphertext outputs: the width rule's
    test on the CPU)"""
    from eva_b200 import EvaProgram, Expr, Input, Output, b200
    from eva_b200._eva_b200 import Type
    from eva_b200.ckks import CKKSCompiler
    prog = EvaProgram("mixed_outputs", 4096)
    with prog:
        x = Input("x")
        p = Expr(prog._make_input("p", Type.Plain), prog)
        r = Input("r", is_encrypted=False)
        Output("y", x * x * p + r)
        Output("z3", Input("x3") + 0.0)
    prog.set_output_ranges(20)
    prog.set_input_scales(30)
    compiled, params, sig = CKKSCompiler().compile(prog)
    pub, sec = b200.generate_keys(params, seed=4)
    pub.set_input_sizes({"x3": 3})
    primes = list(pub.primes())
    N = params.poly_modulus_degree
    rng = np.random.default_rng(6)
    encs = []
    for _ in range(2):
        enc = pub.encrypt({n: list(rng.uniform(0, 1, 4096)) for n in ("x", "p", "r", "x3")}, sig)
        ell = enc.get("x3")[1].shape[1]
        enc.set_cipher("x3", np.stack([[rng.integers(0, int(primes[i]), N, dtype=np.uint64) for i in range(ell)] for _ in range(3)]), 2.0 ** 30)
        encs.append(enc)
    full = pub.execute_batch(compiled, encs)
    assert full[0].get("z3")[0] == "cipher" and full[0].get("z3")[1].shape[0] == 3
    pub.set_options(compact_outputs=10)
    got = pub.execute_batch(compiled, encs)
    assert check_batch(_m(), compiled, primes, full, got, 10, "size 3 next to size 2") == 2
    for f, g in zip(full, got):
        assert g.get("y")[0] == "compact_cipher"
        assert g.get("z3")[0] == "cipher" and np.array_equal(g.get("z3")[1], f.get("z3")[1])


def test_slot_packed_sobel_is_bit_exact():
    from eva_b200 import b200
    from eva_b200.ckks import pack_inputs, pack_program
    d = gl.load_json("sobel")
    prog, params, sig, _ = gl.build_program(d)
    packed, pparams, psig = pack_program(prog, params, sig, 2)
    pub, sec = b200.generate_keys(pparams, seed=12)
    rng = np.random.default_rng(5)
    encs = [sec.encrypt(pack_inputs([{"image": rng.uniform(0, 0.2, sig.vec_size)} for _ in range(2)], sig, 2), psig) for _ in range(2)]
    full = pub.execute_batch(packed, encs)
    pub.set_options(compact_outputs=10)
    assert check_batch(_m(), packed, list(pub.primes()), full, pub.execute_batch(packed, encs), 10, "packed") == 2


def test_server_with_paging_seeded_slots_c1_cache_and_a_stored_input():
    from eva_b200 import b200
    d, prog, params, sig, _, _ = _ctx("sobel")
    ctxs = [b200.generate_keys(params, seed=30 + t) for t in range(3)]
    srv = b200.B200Server(params, capacity=2, max_tenants=3, hoist_constants="inline", key_storage="seeded", c1_cache=1, store_entries=2)
    for p, _ in ctxs:
        srv.add_keys(p)
    encs = [ctxs[t][1].encrypt(client_inputs(d, 50 + t), sig) for t in range(3)]
    stored = request(encs[0], srv.store(0, encs[0]))
    batches = [[(0, stored), (1, encs[1]), (0, stored)], [(2, encs[2]), (1, encs[1])], [(0, stored), (2, encs[2])]]   # 2 slots: pages
    fulls = [srv.execute_batch(prog, rq) for rq in batches]
    built = srv.plans_built()
    srv.set_options(compact_outputs=10)
    primes = list(srv.primes())
    gots = [srv.execute_batch(prog, rq) for rq in batches]
    assert srv.plans_built() == built and srv.bank_info()["evictions"] > 0   # toggling the option built no plan
    for rq, full, got in zip(batches, fulls, gots):
        assert check_batch(_m(), prog, primes, full, got, 10, ("server", [t for t, _ in rq])) == len(rq)
        h = srv.execute_batch_async(prog, rq[::-1], 2)
        check_batch(_m(), prog, primes, full[::-1], srv.execute_batch_result(h), 10, "server async")
        for (t, _), f, c in zip(rq, full, got):
            out, ref = ctxs[t][1].decrypt(c, sig), ctxs[t][1].decrypt(f, sig)
            for n in d["outputs"]:
                assert np.max(np.abs(np.array(out[n]) - np.array(ref[n]))) <= 2.0 ** -10


def test_zero_digit_redo_stays_compact_and_exact():
    """the ciphertext of test_zero_digit_redo_stages_the_stored_input_again: collect's redo compacts with the batch's precision"""
    from eva_b200 import b200
    d = gl.load_json("sobel")
    prog, params, sig, terms = gl.build_program(d)
    N = d["poly_modulus_degree"]
    orc = o.Oracle(N, d["prime_bits"]).keygen(1)
    op = OracleProgram(d, orc)
    op.prepare_keys()
    srv = b200.B200Server(params, capacity=1)
    gks = {int(e): k for e, k in op.gks.items()}
    for e in srv.bank_info()["galois_elements"]:
        gks.setdefault(int(e), orc.galois_key(int(e)))
    t = srv.add_raw_keys(op.rk, gks)
    rng = np.random.default_rng(4)
    (name_, info), = d["signature"].items()
    ell = orc.k - 1 - info["level"]
    ct = orc.encrypt(orc.encode(rng.uniform(0, 1, d["vec_size"]), 2.0 ** info["scale"], ell), seed=3)
    c1 = np.stack([orc.ntt_inv(ct[1, i], i) for i in range(ell)])
    c1[1, 7] = 0
    ct[1] = np.stack([orc.ntt_fwd(c1[i], i) for i in range(ell)])
    val = b200.B200Valuation()
    val.set_cipher(name_, ct, 2.0 ** info["scale"])
    V = op.run({name_: ("cipher", ct, 2.0 ** info["scale"])})
    srv.set_options(compact_outputs=10)
    built = srv.plans_built()
    out = srv.execute(prog, t, val)
    assert srv.plans_built() == built + 2            # the plan, and the one the redo built without the shared mod-up
    srv.set_options(compact_outputs=0, hoist_mod_up=False)
    full = srv.execute(prog, t, val)
    for oname, oid in d["outputs"].items():
        assert np.array_equal(full.get(oname)[1], V[oid][1])
        want = expected_compact(_m(), prog, list(srv.primes()), oname, full.get(oname), 10)
        got = out.get(oname)
        assert got[0] == "compact_cipher" and np.array_equal(got[1], want[0])


# ------------------------------------------------------------------------------------------------ the client
def test_client_integers_equal_exact_decryption():
    d, prog, params, sig, pub, sec = _ctx("polynomial")
    N, primes = d["poly_modulus_degree"], list(pub.primes())
    pub.set_options(compact_outputs=10)
    enc = sec.encrypt(client_inputs(d, 3), sig)
    out = pub.execute(prog, enc)
    sk = sec._export()["secret_key"]
    s = np.array(oracle_for(N, primes).ntt_inv(sk[0], 0), dtype=np.uint64)
    q0 = np.uint64(primes[0])
    sgn = np.where(s == 0, 0, np.where(s == 1, 1, -1)).astype(np.int64)
    assert np.all((s == 0) | (s == 1) | (s == q0 - np.uint64(1)))
    for name in d["outputs"]:
        kind, words, _ = out.get(name)
        assert kind == "compact_cipher"
        b = out.compact_bits(name)
        y0 = np.array(fields(words[0], b, N), dtype=np.uint64)
        y1 = np.array(fields(words[1], b, N), dtype=np.uint64)
        acc = y0.copy()                               # y0 + y1 s mod 2^64 (2^b divides it), negacyclic
        for j in np.nonzero(sgn)[0]:
            r = np.roll(y1, j)
            r[:j] = np.uint64(0) - r[:j]
            acc = acc + r if sgn[j] > 0 else acc - r
        zm = acc & np.uint64((1 << b) - 1)
        z = np.where(zm > np.uint64(1 << (b - 1)), zm.astype(np.int64) - (1 << b), zm.astype(np.int64))
        got = sec.decrypt_compact_poly(words, b)
        assert np.array_equal(got, z)


@pytest.mark.parametrize("p", [8, 16, 24])
def test_decryption_is_within_2_to_minus_p(p):
    from eva_b200 import b200
    d, prog, params, sig, pub, sec = _ctx("sobel")
    encs = [sec.encrypt(client_inputs(d, i), sig) for i in range(4)]
    full = pub.execute_batch(prog, encs)
    pub.set_options(compact_outputs=p)
    comp = pub.execute_batch(prog, encs)
    worst = 0.0
    for f, c in zip(full, comp):
        a, b_ = sec.decrypt(f, sig), sec.decrypt(c, sig)
        for n in d["outputs"]:
            worst = max(worst, float(np.max(np.abs(np.array(a[n]) - np.array(b_[n])))))
    print("compact p=%d: worst |decrypt(compact) - decrypt(full)| = %.3f x 2^-p" % (p, worst * 2.0 ** p))
    assert worst <= 2.0 ** -p


@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_baboon_meets_the_reference_criterion_at_p10(name):
    from eva import evaluate
    from eva.ckks import CKKSCompiler
    from eva.seal import generate_keys
    import tests_programs
    golden = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", GOLDEN))
    inputs = {"image": [x / 255.0 for x in golden["image"].tolist()]}
    expected = golden[name]
    compiled, params, signature = CKKSCompiler().compile(getattr(tests_programs, name)())
    public_ctx, secret_ctx = generate_keys(params)
    public_ctx.set_options(compact_outputs=10)
    res = public_ctx.execute(compiled, secret_ctx.encrypt(inputs, signature))
    assert res.get("image")[0] == "compact_cipher"
    outputs = secret_ctx.decrypt(res, signature)
    assert np.mean((np.array(outputs["image"]) - expected) ** 2) < 0.01


# ------------------------------------------------------------------------------------------------ the value kind (page-locked host buffers)
def test_valuation_and_file_round_trip(tmp_path):
    from eva_b200 import b200, load, save
    N, bits = 1024, 37
    W = (N * bits + 63) // 64
    words = np.random.default_rng(1).integers(0, 2 ** 63, size=(2, W), dtype=np.uint64)
    val = b200.B200Valuation()
    val.set_compact_cipher("out", words, bits, 2.0 ** 20.5)
    kind, arr, scale = val.get("out")
    assert kind == "compact_cipher" and np.array_equal(arr, words) and scale == 2.0 ** 20.5
    assert val.compact_bits("out") == bits
    full = b200.B200Valuation()
    full.set_cipher("out", np.zeros((2, 1, N), dtype=np.uint64), 2.0 ** 25)
    save(val, str(tmp_path / "compact.evab"))
    save(full, str(tmp_path / "full.evab"))
    back = load(str(tmp_path / "compact.evab"))
    kind, arr, scale = back.get("out")
    assert kind == "compact_cipher" and np.array_equal(arr, words) and scale == 2.0 ** 20.5 and back.compact_bits("out") == bits
    assert os.path.getsize(tmp_path / "compact.evab") < 0.6 * os.path.getsize(tmp_path / "full.evab")


def test_compact_bits_of_another_kind_raises():
    from eva_b200 import b200
    val = b200.B200Valuation()
    val.set_cipher("x", np.zeros((2, 1, 1024), dtype=np.uint64), 1.0)
    with pytest.raises(ValueError, match="not a compact ciphertext"):
        val.compact_bits("x")


# ------------------------------------------------------------------------------------------------ the off path, errors
def test_off_path_launches_plans_and_refusals():
    from eva_b200 import b200
    d, prog, params, sig, pub, sec = _ctx("sobel")
    srv = b200.B200Server(params, capacity=1)
    t = srv.add_keys(pub)
    enc = sec.encrypt(client_inputs(d, 1), sig)
    srv.execute(prog, t, enc)
    n0 = srv.launch_count()
    srv.execute(prog, t, enc)
    per_run = srv.launch_count() - n0
    built = srv.plans_built()
    srv.set_options(compact_outputs=20)
    out = srv.execute(prog, t, enc)
    srv.set_options(compact_outputs=0)
    n1 = srv.launch_count()
    full = srv.execute(prog, t, enc)
    assert srv.launch_count() - n1 == per_run and srv.plans_built() == built
    assert full.get("image")[0] == "cipher"
    # a compact value as an input: refused, naming it, before any launch
    bad = b200.B200Valuation()
    kind, words, scale = out.get("image")
    bad.set_compact_cipher("image", words, out.compact_bits("image"), scale)
    n2 = srv.launch_count()
    with pytest.raises(ValueError, match="input image is a compact response"):
        srv.execute(prog, t, bad)
    with pytest.raises(ValueError, match="input image is a compact response"):
        pub.execute(prog, bad)
    assert srv.launch_count() == n2
    with pytest.raises(ValueError, match="compact_outputs"):
        srv.set_options(compact_outputs=53)


def test_compact_call_rejects_bad_arguments():
    from eva_b200 import b200, cabi
    d, prog, params, sig, pub, sec = _ctx("polynomial")
    lib = cabi.load()
    import torch
    be_ctx = C.c_void_p()
    primes = np.array(pub.primes(), dtype=np.uint64)
    assert lib.evab_ctx_create(C.c_uint64(d["poly_modulus_degree"]), primes.ctypes.data_as(u64p), len(primes), 0, C.byref(be_ctx)) == 0
    try:
        buf = torch.zeros(4 * d["poly_modulus_degree"], dtype=torch.int64, device="cuda")
        ptr = buf.data_ptr()
        src = (C.c_void_p * 1)(ptr)
        dst = (C.c_void_p * 1)(ptr + 8 * 2 * d["poly_modulus_degree"])
        work = C.c_void_p(ptr)

        def rejected(rc, word):
            assert rc != 0 and word in lib.evab_last_error().decode(), lib.evab_last_error()
        rejected(lib.evab_compact_ciphers(be_ctx, 1, None, dst, 1, 40, 30, work, None), "h_src")
        rejected(lib.evab_compact_ciphers(be_ctx, 1, src, None, 1, 40, 30, work, None), "h_dst")
        rejected(lib.evab_compact_ciphers(be_ctx, 1, src, dst, 1, 40, 0, work, None), "bits")
        rejected(lib.evab_compact_ciphers(be_ctx, 1, src, dst, 1, 40, 63, work, None), "bits")
        rejected(lib.evab_compact_ciphers(be_ctx, 1, src, dst, 1, 29, 30, work, None), "shift")
        rejected(lib.evab_compact_ciphers(be_ctx, 1, src, dst, 9, 40, 30, work, None), "ell")
        rejected(lib.evab_compact_ciphers(be_ctx, 1, (C.c_void_p * 1)(ptr + 8), dst, 1, 40, 30, work, None), "h_src[0]")
        rejected(lib.evab_compact_ciphers(be_ctx, 1, src, (C.c_void_p * 1)(ptr + 4), 1, 40, 30, work, None), "h_dst[0]")
        rejected(lib.evab_compact_ciphers(be_ctx, 1, src, dst, 1, 40, 30, C.c_void_p(ptr + 8), None), "d_work")
        torch.cuda.synchronize()
    finally:
        lib.evab_ctx_destroy(be_ctx)
