"""Seed-compressed input ciphertexts on the GPU: evab_expand_cipher_uniform against the CPU replay, secret-key encryption checked
exactly with the oracle NTT, seeded inputs giving the same output bytes as the same ciphertexts in full on every execution path,
the round trip against the reference's plaintext results, files, and the error cases."""
import ctypes as C

import numpy as np
import pytest

from backends import GpuBackend
from oracle import oracle as o
from test_compressed_keys import HIGH_REJECTION, seeds_for
from test_compressed_keys_gpu import _same
from test_seeded_inputs import SENTINEL, np_cipher_c1, replay_cipher

pytestmark = pytest.mark.gpu
u64p = C.POINTER(C.c_uint64)


def expand_args(seeds, ptrs, ells, moduli):
    n = len(seeds)
    return (C.c_char_p(b"".join(seeds)), (C.c_void_p * n)(*ptrs), (C.c_int * n)(*ells), np.array(moduli, dtype=np.uint64))


def device_expand(N, primes, moduli, seeds, ells, guard=64):
    """one device buffer holding a ciphertext [2][ell_i][N] per entry (then `guard` words), all at a sentinel; returns the buffer
    after the expansion, split per entry, and checks that only the c1 rows were written"""
    be = GpuBackend(N, primes)
    sizes = [2 * ell * N for ell in ells]
    total = sum(sizes) + guard
    d = be._up(np.full(total, SENTINEL, dtype=np.uint64))
    offs = np.cumsum([0] + sizes[:-1])
    ptrs = [d.value + 8 * (int(off) + ell * N) for off, ell in zip(offs, ells)]
    sd, pp, el, qa = expand_args(seeds, ptrs, ells, moduli)
    be._chk(be.lib.evab_expand_cipher_uniform(be.h, len(seeds), sd, pp, el, qa.ctypes.data_as(u64p), None))
    got = be._down(d, (total,))
    be._free(d)
    assert (got[sum(sizes):] == SENTINEL).all()
    cts = [got[off:off + s].reshape(2, ell, N) for off, s, ell in zip(offs, sizes, ells)]
    for ct in cts:
        assert (ct[0] == SENTINEL).all()
    return [ct[1] for ct in cts]


@pytest.mark.parametrize("N,bits,ells", [(16384, [60] * 5, [1, 2, 3, 4, 4, 2]), (32768, [60] * 14, [13, 7])])
def test_device_expansion_equals_replay(N, bits, ells):
    primes = o.gen_primes(N, bits)
    seeds = seeds_for(len(ells), N + len(bits))
    got = device_expand(N, primes, primes, seeds, ells)
    want = replay_cipher(seeds, ells, N, primes)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    if N == 16384:
        assert np.array_equal(got[3], np_cipher_c1(seeds[3], N, primes, 4)[0])


def test_device_expansion_high_rejection_moduli():
    N = 16384
    primes = o.gen_primes(N, [60] * 4)
    seeds = seeds_for(2, 19)
    got = device_expand(N, primes, HIGH_REJECTION, seeds, [3, 2])
    want, fell = np_cipher_c1(seeds[0], N, HIGH_REJECTION, 3)
    assert (fell > 0).all() and np.array_equal(got[0], want)
    assert np.array_equal(got[1], replay_cipher(seeds[1:], [2], N, HIGH_REJECTION)[0])


def test_device_expansion_more_entries_than_one_launch():
    """200 entries (several launches of at most 56) give the words of the replay"""
    N = 4096
    primes = o.gen_primes(N, [60] * 4)
    seeds = seeds_for(200, 23)
    ells = [1 + i % 3 for i in range(200)]
    for g, w in zip(device_expand(N, primes, primes, seeds, ells), replay_cipher(seeds, ells, N, primes)):
        assert np.array_equal(g, w)


def test_device_expansion_rejects_bad_arguments():
    N = 1024
    primes = o.gen_primes(N, [60] * 3)
    be = GpuBackend(N, primes)
    d = be._up(np.zeros(8 * N, dtype=np.uint64))
    sd, pp, el, qa = expand_args([bytes(32)], [d.value + 8 * N], [1], primes)
    q = qa.ctypes.data_as(u64p)
    f = be.lib.evab_expand_cipher_uniform

    def rejected(rc, word):
        assert rc != 0 and word in be.lib.evab_last_error(), be.lib.evab_last_error()

    rejected(f(be.h, 0, sd, pp, el, q, None), b"n must be")
    rejected(f(be.h, 65536, sd, pp, el, q, None), b"n must be")
    rejected(f(be.h, 1, None, pp, el, q, None), b"h_seeds")
    rejected(f(be.h, 1, sd, None, el, q, None), b"h_c1")
    rejected(f(be.h, 1, sd, pp, None, q, None), b"h_ell")
    rejected(f(be.h, 1, sd, pp, el, None, None), b"h_moduli")
    rejected(f(be.h, 1, sd, (C.c_void_p * 1)(None), el, q, None), b"h_c1[0]")
    for bad in (0, 3):                                   # k = 3: ell in [1, 2]
        rejected(f(be.h, 1, sd, pp, (C.c_int * 1)(bad), q, None), b"h_ell[0]")
    qa[0] = 1
    rejected(f(be.h, 1, sd, pp, el, q, None), b"modulus")
    be._free(d)


# --------------------------------------------------------------------------------------------------------- secret-key encryption
def _ctx(name, seed=5):
    from eva_b200 import b200, program_io as gl
    d = gl.load_json(name)
    prog, params, sig, _ = gl.build_program(d)
    pub, sec = b200.generate_keys(params, seed=seed)
    return d, prog, params, sig, pub, sec


def test_seeded_encryption_is_exact():
    """c1 is the seed's expansion, and c0 + c1 s - pt = -NTT(e) mod q_m on every row"""
    d, prog, params, sig, pub, sec = _ctx("polynomial")
    sk = sec._export()["secret_key"]
    N, primes = d["poly_modulus_degree"], list(pub.primes())
    orc = o.Oracle(N, primes=primes)
    rng = np.random.default_rng(3)
    for ell in range(1, len(primes)):
        pt = pub.encode(list(rng.uniform(-1, 1, N // 2)), 2.0 ** 30, ell)
        seed = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
        e = [int(x) for x in rng.integers(-21, 22, N)]
        ct = sec.encrypt_seeded_poly(pt, seed, e)
        assert np.array_equal(ct, pub.encrypt_seeded_poly(pt, seed, e))     # same client, same secret
        assert np.array_equal(ct[1], replay_cipher([seed], [ell], N, primes)[0])
        for m in range(ell):
            q = primes[m]
            v = (ct[0, m].astype(object) + ct[1, m].astype(object) * sk[m].astype(object) - pt[m].astype(object)) % q
            got = orc.ntt_inv(np.array(v, dtype=np.uint64), m).astype(object)
            assert all(int(g) == (-x) % q for g, x in zip(got, e)), (ell, m)
    with pytest.raises(Exception, match="32 bytes"):
        sec.encrypt_seeded_poly(pt, seed[:31], e)


def _plain_program():
    from eva_b200 import EvaProgram, Expr, Input, Output
    from eva_b200._eva_b200 import Type
    from eva_b200.ckks import CKKSCompiler
    prog = EvaProgram("plain_input", 64)
    with prog:
        x = Input("x")
        p = Expr(prog._make_input("p", Type.Plain), prog)
        r = Input("r", is_encrypted=False)
        Output("y", x * p + r)
    prog.set_output_ranges(30)
    prog.set_input_scales(30)
    return CKKSCompiler().compile(prog)


def test_secret_encrypt_makes_seeded_ciphers_and_public_plains():
    from eva_b200 import b200
    prog, params, sig = _plain_program()
    pub, sec = b200.generate_keys(params, seed=9)
    rng = np.random.default_rng(1)
    inputs = {n: list(rng.uniform(0, 1, 64)) for n in ("x", "p", "r")}
    a, b = sec.encrypt(inputs, sig), pub.encrypt(inputs, sig)
    kind, c0, scale = a.get("x")
    assert kind == "seeded_cipher" and c0.shape == (len(params.prime_bits) - 1, params.poly_modulus_degree) and scale == 2.0 ** 30
    assert b.get("x")[0] == "cipher"
    for n in ("p", "r"):        # Plain and Raw inputs as the public path makes them
        assert a.get(n)[0] == b.get(n)[0] and np.array_equal(np.asarray(a.get(n)[1]), np.asarray(b.get(n)[1])) and a.get(n)[2] == b.get(n)[2]
    # a fresh seed per ciphertext
    seeds = {sec.encrypt(inputs, sig).get_seed("x") for _ in range(4)} | {a.get_seed("x")}
    assert len(seeds) == 5 and all(len(s) == 32 for s in seeds)
    out = sec.decrypt(pub.execute(prog, a), sig)["y"]
    want = np.array(inputs["x"]) * np.array(inputs["p"]) + np.array(inputs["r"])
    assert np.abs(np.array(out) - want).max() < 1e-3
    assert not hasattr(pub, "encrypt_seeded")


# ------------------------------------------------------------------------------------------------ seeded == full, every path
def full_of(val, N, primes):
    """the same valuation with every seeded ciphertext in full: c0 and its c1 replayed on the CPU"""
    from eva_b200 import b200
    out = b200.B200Valuation()
    for n in val.names():
        kind, arr, scale = val.get(n)
        if kind == "seeded_cipher":
            c1 = replay_cipher([val.get_seed(n)], [arr.shape[0]], N, primes)[0]
            out.set_cipher(n, np.ascontiguousarray(np.stack([arr, c1])), scale)
        elif kind == "cipher":
            out.set_cipher(n, arr, scale)
        elif kind == "plain":
            out.set_plain(n, arr, scale)
        else:
            out.set_raw(n, list(arr))
    return out


def client_inputs(d, i):
    rng = np.random.default_rng(700 + i)
    return {n: list(rng.uniform(0.0, 0.2, d["vec_size"])) for n in d["signature"]}


def _outs(vals, d):
    return [{n: v.get(n) for n in d["outputs"]} for v in vals]


@pytest.mark.parametrize("name", ["sobel", "harris", "feat_mixed"])
def test_seeded_and_full_inputs_give_the_same_bytes(name):
    from eva_b200 import b200
    d, prog, params, sig, pub, sec = _ctx(name)
    N, primes = d["poly_modulus_degree"], list(pub.primes())
    B = 32
    seeded = [sec.encrypt(client_inputs(d, i), sig) for i in range(B)]
    full = [full_of(v, N, primes) for v in seeded]
    assert all(v.get(n)[0] == "seeded_cipher" for v in seeded for n in v.names() if d["signature"][n]["type"] == "Cipher")
    want = _outs(pub.execute_batch(prog, full), d)
    _same(_outs([pub.execute(prog, seeded[0])], d), want[:1], (name, "execute"))
    mixed = [seeded[i] if i % 2 else full[i] for i in range(B)]
    _same(_outs(pub.execute_batch(prog, mixed), d), want, (name, "execute_batch mixed"))
    h0 = pub.execute_batch_async(prog, seeded, 0)
    h1 = pub.execute_batch_async(prog, mixed[::-1], 1)
    _same(_outs(pub.execute_batch_result(h0), d), want, (name, "async"))
    _same(_outs(pub.execute_batch_result(h1), d), want[::-1], (name, "async reversed"))
    # one fused chunk of 32 instances: one expansion call for all of its seeded inputs
    pub.set_options(fuse=B)
    _same(_outs(pub.execute_batch(prog, mixed), d), want, (name, "execute_batch fused"))
    pub.set_options()
    # server, resident: three clients, each with its own keys and its own seeded inputs
    clients = [(pub, sec)] + [b200.generate_keys(params, seed=s) for s in (6, 7)]
    vals = [seeded[:4]] + [[c[1].encrypt(client_inputs(d, 40 + 4 * t + i), sig) for i in range(4)] for t, c in enumerate(clients[1:])]
    fulls = [[full_of(v, N, primes) for v in row] for row in vals]
    srv = b200.B200Server(params, capacity=3)
    for c in clients:
        srv.add_keys(c[0])

    def run(server, assign, src):
        return _outs(server.execute_batch(prog, [(t, src[t][i]) for i, t in enumerate(assign)]), d)
    for a in ([0, 1, 2, 0], [2, 2, 1, 0]):
        _same(run(srv, a, vals), run(srv, a, fulls), (name, "server", a))
    # server, paged with evictions (2 slots, 3 tenants)
    paged = b200.B200Server(params, capacity=2, max_tenants=4)
    for c in clients:
        paged.add_keys(c[0])
    for a in ([2, 2, 2, 2], [0, 1, 0, 1], [1, 2, 2, 1], [0, 0, 0, 0], [2, 0, 0, 2]):
        _same(run(paged, a, vals), run(srv, a, fulls), (name, "paged", a))
    assert paged.bank_info()["evictions"] > 0


def test_device_resident_hooks_stage_seeded_inputs():
    import torch
    from eva_b200 import b200
    d, prog, params, sig, pub, sec = _ctx("sobel")
    N, primes = d["poly_modulus_degree"], list(pub.primes())
    v = sec.encrypt(client_inputs(d, 0), sig)
    f = full_of(v, N, primes)
    st = torch.cuda.Stream()
    outs = []
    for val in (v, f):
        pub.stage_inputs(prog, [val], st.cuda_stream, 0)
        pub.run_resident(prog, st.cuda_stream, 1, 0)
        outs.append(_outs([pub.download_outputs(prog, st.cuda_stream, 0)], d))
    _same(outs[0], outs[1], "resident hooks")
    srv = b200.B200Server(params, capacity=2)
    srv.add_keys(pub)
    got = []
    for val in (v, f):
        srv.stage_inputs(prog, [(0, val), (0, val)], st.cuda_stream, 0)
        srv.run_resident(prog, st.cuda_stream, 2, 0)
        st.synchronize()
        got.append([srv.debug_value(prog, prog.outputs[n].index, 2, b)[0] for n in d["outputs"] for b in range(2)])
    assert all(np.array_equal(x, y) for x, y in zip(*got))


# ------------------------------------------------------------------------------------------------------- round trip, files
GOLDEN = "image_processing_baboon.npz"


@pytest.mark.parametrize("name", ["sobel", "harris"])
def test_round_trip_meets_the_reference_criterion(name):
    import os
    from eva import evaluate
    from eva.ckks import CKKSCompiler
    from eva.seal import generate_keys
    import tests_programs
    golden = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", GOLDEN))
    inputs = {"image": [x / 255.0 for x in golden["image"].tolist()]}
    expected = golden[name]
    compiled, params, signature = CKKSCompiler().compile(getattr(tests_programs, name)())
    assert np.mean((np.array(evaluate(compiled, inputs)["image"]) - expected) ** 2) < 1e-10
    public_ctx, secret_ctx = generate_keys(params)
    enc = secret_ctx.encrypt(inputs, signature)
    assert enc.get("image")[0] == "seeded_cipher"
    outputs = secret_ctx.decrypt(public_ctx.execute(compiled, enc), signature)
    assert np.mean((np.array(outputs["image"]) - expected) ** 2) < 0.01


def test_client_server_flow_through_files(tmp_path):
    """secret context, public context and a seeded valuation cross files; the server's bytes equal the in-memory flow's"""
    from eva_b200 import load, save
    d, prog, params, sig, pub, sec = _ctx("sobel", seed=0)
    enc = sec.encrypt(client_inputs(d, 1), sig)
    want = _outs([pub.execute(prog, enc)], d)
    save(sec, str(tmp_path / "c.sealsecret"))
    save(pub, str(tmp_path / "s.sealpublic"))
    save(enc, str(tmp_path / "in.sealvals"))
    sec2, pub2, enc2 = load(str(tmp_path / "c.sealsecret")), load(str(tmp_path / "s.sealpublic")), load(str(tmp_path / "in.sealvals"))
    assert enc2.get("image")[0] == "seeded_cipher" and enc2.get_seed("image") == enc.get_seed("image")
    assert np.array_equal(enc2.get("image")[1], enc.get("image")[1])
    res = pub2.execute(prog, enc2)
    _same(_outs([res], d), want, "through files")
    a = sec2.decrypt(res, sig)["image"]
    b = sec.decrypt(pub.execute(prog, enc), sig)["image"]
    assert np.array_equal(np.array(a), np.array(b))
    # a loaded secret context encrypts seeded inputs too (fresh OS-entropy seeds and errors), and they decrypt to the same result
    # within the reference's criterion
    enc3 = sec2.encrypt(client_inputs(d, 1), sig)
    assert enc3.get_seed("image") != enc.get_seed("image")
    assert np.mean((np.array(sec.decrypt(pub2.execute(prog, enc3), sig)["image"]) - np.array(b)) ** 2) < 0.01


def test_seeded_valuation_serializes_at_half_the_size():
    from eva_b200 import b200, serialization as ser
    N, ell = 16384, 4
    rng = np.random.default_rng(2)
    c0 = rng.integers(0, 1 << 59, (ell, N), dtype=np.uint64)
    c1 = rng.integers(0, 1 << 59, (ell, N), dtype=np.uint64)
    seed = bytes(range(32))
    v = b200.B200Valuation()
    v.set_seeded_cipher("image", c0, seed, 2.0 ** 25)
    v.set_raw("r", [1.0, 2.0])
    w = b200.B200Valuation()
    w.set_cipher("image", np.stack([c0, c1]), 2.0 ** 25)
    w.set_raw("r", [1.0, 2.0])
    blob, full_blob = ser.dumps(v), ser.dumps(w)
    assert 0.49 < len(blob) / len(full_blob) < 0.51, (len(blob), len(full_blob))
    back = ser.loads(blob)
    kind, arr, scale = back.get("image")
    assert kind == "seeded_cipher" and np.array_equal(arr, c0) and scale == 2.0 ** 25 and back.get_seed("image") == seed
    assert back.get("r")[1] == [1.0, 2.0]
    again = ser.loads(full_blob)
    assert again.get("image")[0] == "cipher" and np.array_equal(again.get("image")[1], np.stack([c0, c1]))
    # shard subsets carry the kind across
    from eva_b200 import dagshard, shard
    for mod in (shard, dagshard):
        sub = mod._subset(v, {"image"})
        assert sub.names() == ["image"] and sub.get("image")[0] == "seeded_cipher" and sub.get_seed("image") == seed


# ------------------------------------------------------------------------------------------------------------------ errors
def test_seeded_inputs_are_checked():
    from eva_b200 import b200
    d, prog, params, sig, pub, sec = _ctx("sobel")
    enc = sec.encrypt(client_inputs(d, 2), sig)
    _, c0, scale = enc.get("image")
    seed = enc.get_seed("image")

    def one(arr, s=seed):
        v = b200.B200Valuation()
        v.set_seeded_cipher("image", np.ascontiguousarray(arr), s, scale)
        return v
    with pytest.raises(Exception, match="does not match"):
        pub.execute(prog, one(c0[:-1]))                             # wrong ell
    with pytest.raises(Exception, match="does not match"):
        pub.execute(prog, one(c0[:, : c0.shape[1] // 2]))           # wrong N
    with pytest.raises(Exception, match="32 bytes"):
        one(c0, seed[:31])
    with pytest.raises(Exception, match=r"\[ell\]\[N\]"):
        b200.B200Valuation().set_seeded_cipher("image", c0[None], seed, scale)
    with pytest.raises(Exception, match="not a seeded ciphertext"):
        pub.encrypt(client_inputs(d, 2), sig).get_seed("image")
    pprog, pparams, psig = _plain_program()
    ppub, psec = b200.generate_keys(pparams, seed=4)
    good = psec.encrypt({n: [0.5] * 64 for n in ("x", "p", "r")}, psig)
    # declared size 3 (x * p + r takes one): a seeded ciphertext is always size 2
    ppub.set_input_sizes({"x": 3})
    with pytest.raises(Exception, match="input x: seeded ciphertext does not match"):
        ppub.execute(pprog, good)
    ppub.set_input_sizes({})
    ppub.drop_plan(pprog)
    # a seeded value for a Plain input
    bad = b200.B200Valuation()
    bad.set_seeded_cipher("x", good.get("x")[1], good.get_seed("x"), good.get("x")[2])
    bad.set_seeded_cipher("p", good.get("x")[1], good.get_seed("x"), good.get("p")[2])
    bad.set_raw("r", [0.5] * 64)
    with pytest.raises(Exception, match="input p: seeded ciphertext does not match"):
        ppub.execute(pprog, bad)
    # the valid inputs still run after the errors
    _same(_outs([pub.execute(prog, enc)], d), _outs([pub.execute(prog, full_of(enc, d["poly_modulus_degree"], list(pub.primes())))], d), "after errors")
