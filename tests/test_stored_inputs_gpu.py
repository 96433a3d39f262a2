"""Server-resident ciphertexts on the GPU: a request that names a stored entry by handle gives the same output bytes as the same
ciphertext sent inline, on every execution path and server variant; evab_gather_ciphers on its own; and every error path, none of
which issues a launch."""
import ctypes as C

import numpy as np
import pytest

from backends import GpuBackend
from eva_b200 import program_io as gl
from oracle import oracle as o
from oracle_exec import OracleProgram
from test_compressed_keys_gpu import _same
from test_seeded_inputs_gpu import _ctx, _outs, client_inputs

pytestmark = pytest.mark.gpu
u64p = C.POINTER(C.c_uint64)
SENTINEL = 0xA5A5A5A5A5A5A5A5


def copy_value(src, dst, name):
    kind, arr, scale = src.get(name)
    if kind == "cipher":
        dst.set_cipher(name, arr, scale)
    elif kind == "seeded_cipher":
        dst.set_seeded_cipher(name, arr, src.get_seed(name), scale)
    elif kind == "plain":
        dst.set_plain(name, arr, scale)
    elif kind == "stored":
        dst.set_stored(name, arr)
    else:
        dst.set_raw(name, list(arr))


def request(val, handles):
    """`val` without the names in `handles`, and a reference to each handle's stored entry"""
    from eva_b200 import b200
    out = b200.B200Valuation()
    for n in val.names():
        if n not in handles:
            copy_value(val, out, n)
    for n, h in handles.items():
        out.set_stored(n, h)
    return out


def encrypt_with(pub, sec, storage, inputs, sig):
    return (sec.encrypt if storage == "seeded" else pub.encrypt)(inputs, sig)


# ------------------------------------------------------------------------------------------------------------ every path, Sobel
@pytest.mark.parametrize("storage", ["full", "seeded"])
def test_sobel_stored_image_equals_inline(storage):
    import torch
    from eva_b200 import b200
    d, prog, params, sig, pub, sec = _ctx("sobel")
    B = 32
    srv = b200.B200Server(params, capacity=2, store_entries=B + 1)
    t = srv.add_keys(pub)
    encs = [encrypt_with(pub, sec, storage, client_inputs(d, i), sig) for i in range(B)]
    want = _outs(srv.execute_batch(prog, [(t, e) for e in encs]), d)
    handles = [srv.store(t, e) for e in encs]
    assert all(list(h) == ["image"] for h in handles)
    ids = [h["image"] for h in handles]
    assert ids == sorted(ids) and len(set(ids)) == B
    info = srv.bank_info()
    assert info["store_entries"] == B + 1 and info["stored"] == B
    assert info["store_entry_bytes"] == 2 * (len(params.prime_bits) - 1) * params.poly_modulus_degree * 8
    assert info["store_bytes"] == (B + 1) * info["store_entry_bytes"]
    reqs = [request(e, h) for e, h in zip(encs, handles)]
    assert reqs[0].get("image") == ("stored", ids[0], None)
    _same(_outs([srv.execute(prog, t, reqs[0])], d), want[:1], (storage, "execute"))
    _same(_outs(srv.execute_batch(prog, [(t, r) for r in reqs]), d), want, (storage, "execute_batch"))
    mixed = [(t, reqs[i] if i % 2 else encs[i]) for i in range(B)]
    h0 = srv.execute_batch_async(prog, [(t, r) for r in reqs], 0)
    h1 = srv.execute_batch_async(prog, mixed[::-1], 1)
    _same(_outs(srv.execute_batch_result(h0), d), want, (storage, "async"))
    _same(_outs(srv.execute_batch_result(h1), d), want[::-1], (storage, "async mixed reversed"))
    srv.set_options(fuse=B)                        # one chunk of 32: one gather for all of its stored inputs
    _same(_outs(srv.execute_batch(prog, mixed), d), want, (storage, "fused"))
    srv.set_options()
    st = torch.cuda.Stream()
    got = []
    for pair in ((reqs[0], reqs[1]), (encs[0], encs[1])):
        srv.stage_inputs(prog, [(t, pair[0]), (t, pair[1])], st.cuda_stream, 0)
        srv.run_resident(prog, st.cuda_stream, 2, 0)
        st.synchronize()
        got.append([srv.debug_value(prog, prog.outputs[n].index, 2, b)[0] for n in d["outputs"] for b in range(2)])
    assert all(np.array_equal(x, y) for x, y in zip(*got))
    for i in ids:
        srv.release(i)
    assert srv.bank_info()["stored"] == 0


def test_two_cipher_inputs_one_stored_one_inline():
    from eva_b200 import b200
    d, prog, params, sig, pub, sec = _ctx("feat_bin_mul_11")
    srv = b200.B200Server(params, capacity=1, store_entries=4)
    t = srv.add_keys(pub)
    encs = [pub.encrypt(client_inputs(d, i), sig) for i in range(4)]
    want = _outs(srv.execute_batch(prog, [(t, e) for e in encs]), d)
    reqs = []
    for i, e in enumerate(encs):                   # a stored in even requests, b in odd ones
        name = "ab"[i % 2]
        one = b200.B200Valuation()
        copy_value(e, one, name)
        reqs.append(request(e, srv.store(t, one)))
    _same(_outs(srv.execute_batch(prog, [(t, r) for r in reqs]), d), want, "one stored, one inline")


def test_one_handle_named_by_several_instances():
    from eva_b200 import b200
    d, prog, params, sig, pub, sec = _ctx("sobel")
    other, _ = b200.generate_keys(params, seed=8)
    srv = b200.B200Server(params, capacity=2, store_entries=2)
    t0, t1 = srv.add_keys(pub), srv.add_keys(other)
    shared = pub.encrypt(client_inputs(d, 0), sig)
    h = srv.store(t0, shared)
    inline1 = other.encrypt(client_inputs(d, 1), sig)
    rq = [(t0, request(shared, h)), (t1, inline1), (t0, request(shared, h)), (t0, shared), (t1, inline1), (t0, request(shared, h))]
    want = _outs(srv.execute_batch(prog, [(t, shared if t == t0 else inline1) for t, _ in rq]), d)
    _same(_outs(srv.execute_batch(prog, rq), d), want, "shared handle")
    srv.set_options(fuse=len(rq))
    _same(_outs(srv.execute_batch(prog, rq), d), want, "shared handle, one chunk")


# ------------------------------------------------------------------------------------------------------------- server variants
def test_paging_server_keeps_entries_while_keys_move():
    from eva_b200 import b200
    d, prog, params, sig, _, _ = _ctx("sobel")
    pubs = [b200.generate_keys(params, seed=20 + t)[0] for t in range(3)]
    srv = b200.B200Server(params, capacity=2, max_tenants=3, store_entries=3)
    ref = b200.B200Server(params, capacity=3)
    for p in pubs:
        srv.add_keys(p)
        ref.add_keys(p)
    encs = [pubs[t].encrypt(client_inputs(d, 10 + t), sig) for t in range(3)]
    handles = [srv.store(t, encs[t]) for t in range(3)]
    for order in ([0], [1, 2], [0, 0], [2], [1, 0, 1], [2, 0]):
        got = srv.execute_batch(prog, [(t, request(encs[t], handles[t])) for t in order])
        _same(_outs(got, d), _outs(ref.execute_batch(prog, [(t, encs[t]) for t in order]), d), ("paged", order))
    assert srv.bank_info()["evictions"] > 0 and srv.bank_info()["stored"] == 3


def test_seeded_bank_with_c1_cache():
    from eva_b200 import b200
    d, prog, params, sig, _, _ = _ctx("sobel")
    ctxs = [b200.generate_keys(params, seed=30 + t) for t in range(2)]
    srv = b200.B200Server(params, capacity=2, hoist_constants="inline", key_storage="seeded", c1_cache=1, store_entries=4)
    for p, _ in ctxs:
        srv.add_keys(p)
    encs = [ctxs[t][1].encrypt(client_inputs(d, 40 + t), sig) for t in range(2)]
    handles = [srv.store(t, encs[t]) for t in range(2)]
    order = [0, 1, 1, 0]
    want = _outs(srv.execute_batch(prog, [(t, encs[t]) for t in order]), d)
    _same(_outs(srv.execute_batch(prog, [(t, request(encs[t], handles[t])) for t in order]), d), want, "seeded c1 cache")


def test_slot_packed_program():
    from eva_b200 import b200
    from eva_b200.ckks import pack_inputs, pack_program
    d = gl.load_json("sobel")
    prog, params, sig, _ = gl.build_program(d)
    packed, pparams, psig = pack_program(prog, params, sig, 2)
    pub, sec = b200.generate_keys(pparams, seed=12)
    srv = b200.B200Server(pparams, capacity=1, store_entries=2)
    t = srv.add_keys(pub)
    rng = np.random.default_rng(5)
    encs = [sec.encrypt(pack_inputs([{"image": rng.uniform(0, 0.2, sig.vec_size)} for _ in range(2)], sig, 2), psig) for _ in range(2)]
    want = _outs(srv.execute_batch(packed, [(t, e) for e in encs]), d)
    _same(_outs(srv.execute_batch(packed, [(t, request(e, srv.store(t, e))) for e in encs]), d), want, "packed k = 2")


def test_zero_digit_redo_stages_the_stored_input_again():
    """the ciphertext of test_zero_digit_falls_back_to_the_exact_path, stored: collect's redo gathers it again and returns the oracle's bits"""
    from eva_b200 import b200
    d = gl.load_json("sobel")
    prog, params, sig, terms = gl.build_program(d)
    N = d["poly_modulus_degree"]
    orc = o.Oracle(N, d["prime_bits"]).keygen(1)
    op = OracleProgram(d, orc)
    op.prepare_keys()
    srv = b200.B200Server(params, capacity=1, store_entries=1)
    assert list(srv.primes()) == list(orc.primes)
    gks = {int(e): k for e, k in op.gks.items()}
    for e in srv.bank_info()["galois_elements"]:    # the server's set also holds step 0's element, which no rotation reads
        gks.setdefault(int(e), orc.galois_key(int(e)))
    t = srv.add_raw_keys(op.rk, gks)
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
    req = request(val, srv.store(t, val))
    built = srv.plans_built()
    out = srv.execute(prog, t, req)
    assert srv.plans_built() == built + 2            # the plan, and the one the redo built without the shared mod-up
    for oname, oid in d["outputs"].items():
        assert np.array_equal(out.get(oname)[1], V[oid][1])


# ------------------------------------------------------------------------------------------------------ evab_gather_ciphers
def _gather(be, srcs, dsts, words):
    n = len(srcs)
    w = np.array(words, dtype=np.uint64)
    return be.lib.evab_gather_ciphers(be.h, n, (C.c_void_p * max(n, 1))(*srcs), (C.c_void_p * max(n, 1))(*dsts), w.ctypes.data_as(u64p), None)


def test_gather_more_entries_than_one_launch_leaves_guards():
    """400 entries of mixed lengths (three launches of at most 160), each destination between sentinel guards"""
    N = 1024
    be = GpuBackend(N, o.gen_primes(N, [60] * 3))
    rng = np.random.default_rng(0)
    n, guard = 400, 2
    words = [2 * int(x) for x in rng.integers(1, 1200, n)]
    src = rng.integers(0, 2 ** 63, sum(words), dtype=np.uint64)
    d_src = be._up(src)
    total = sum(w + guard for w in words) + guard
    d_dst = be._up(np.full(total, SENTINEL, dtype=np.uint64))
    soff = np.cumsum([0] + words[:-1])
    doff = [guard + sum(w + guard for w in words[:i]) for i in range(n)]
    l0 = be.lib.evab_launch_count(be.h)
    be._chk(_gather(be, [d_src.value + 8 * int(s) for s in soff], [d_dst.value + 8 * x for x in doff], words))
    assert be.lib.evab_launch_count(be.h) - l0 == 3
    got = be._down(d_dst, (total,))
    mask = np.ones(total, dtype=bool)
    for s, x, w in zip(soff, doff, words):
        assert np.array_equal(got[x:x + w], src[s:s + w])
        mask[x:x + w] = False
    assert (got[mask] == SENTINEL).all()
    be._chk(_gather(be, [], [], []))                 # n = 0: nothing to do, no launch
    assert be.lib.evab_launch_count(be.h) - l0 == 3
    be._free(d_src)
    be._free(d_dst)


def test_gather_rejects_bad_arguments():
    N = 1024
    be = GpuBackend(N, o.gen_primes(N, [60] * 3))
    d = be._up(np.zeros(64, dtype=np.uint64))
    f = be.lib.evab_gather_ciphers
    ok_src, ok_dst = (C.c_void_p * 1)(d.value), (C.c_void_p * 1)(d.value + 256)
    w = np.array([8], dtype=np.uint64)
    wp = w.ctypes.data_as(u64p)
    l0 = be.lib.evab_launch_count(be.h)

    def rejected(rc, word):
        assert rc != 0 and word in be.lib.evab_last_error(), be.lib.evab_last_error()
    rejected(f(be.h, -1, ok_src, ok_dst, wp, None), b"n must be")
    rejected(f(be.h, 1, None, ok_dst, wp, None), b"h_src is null")
    rejected(f(be.h, 1, ok_src, None, wp, None), b"h_dst is null")
    rejected(f(be.h, 1, ok_src, ok_dst, None, None), b"h_words is null")
    rejected(f(be.h, 1, (C.c_void_p * 1)(d.value + 8), ok_dst, wp, None), b"h_src[0]")
    rejected(f(be.h, 1, (C.c_void_p * 1)(None), ok_dst, wp, None), b"h_src[0]")
    rejected(f(be.h, 1, ok_src, (C.c_void_p * 1)(d.value + 264), wp, None), b"h_dst[0]")
    rejected(f(be.h, 1, ok_src, (C.c_void_p * 1)(None), wp, None), b"h_dst[0]")
    rejected(f(be.h, 1, ok_src, ok_dst, np.array([7], dtype=np.uint64).ctypes.data_as(u64p), None), b"h_words[0]")
    assert be.lib.evab_launch_count(be.h) == l0
    be._free(d)


# ------------------------------------------------------------------------------------------------------------------- errors
def test_errors_name_the_input_and_issue_no_launch():
    from eva_b200 import b200
    d, prog, params, sig, pub, sec = _ctx("sobel")
    other, _ = b200.generate_keys(params, seed=77)
    srv = b200.B200Server(params, capacity=2, store_entries=2)
    a, b = srv.add_keys(pub), srv.add_keys(other)
    enc = pub.encrypt(client_inputs(d, 3), sig)
    h = srv.store(a, enc)["image"]
    srv.execute_batch(prog, [(a, enc), (a, enc)])    # plans built: what follows measures launches only
    srv.execute(prog, a, enc)

    def refused(fn, *words):
        before = srv.launch_count()
        with pytest.raises(Exception) as e:
            fn()
        for w in words:
            assert w in str(e.value), (w, str(e.value))
        assert srv.launch_count() == before
    ref = b200.B200Valuation()
    ref.set_stored("image", h)
    refused(lambda: srv.execute_batch(prog, [(a, enc), (b, ref)]), "input image", "handle %d" % h, "tenant %d" % b, "another tenant")
    refused(lambda: srv.execute(prog, b, ref), "handle %d" % h, "tenant %d" % b)
    # a level that does not match the plan's: the same ciphertext one prime lower
    low = b200.B200Valuation()
    _, ct, scale = enc.get("image")
    low.set_cipher("image", np.ascontiguousarray(ct[:, :-1]), scale)
    hl = srv.store(a, low)["image"]
    bad = b200.B200Valuation()
    bad.set_stored("image", hl)
    refused(lambda: srv.execute_batch(prog, [(a, ref), (a, bad)]), "input image", "handle %d" % hl, "tenant %d" % a, "does not match")
    # full store (2 entries in use), and plain / raw values: nothing stored
    refused(lambda: srv.store(a, enc), "store_entries=2")
    srv.release(hl)
    plain = b200.B200Valuation()
    copy_value(enc, plain, "image")
    plain.set_raw("r", [1.0])
    refused(lambda: srv.store(a, plain), "value r")
    assert srv.bank_info()["stored"] == 1
    # released handle
    refused(lambda: srv.release(hl), "handle %d" % hl)
    gone = b200.B200Valuation()
    gone.set_stored("image", hl)
    refused(lambda: srv.execute(prog, a, gone), "handle %d" % hl, "no such entry")
    # release and remove_keys while an uncollected batch names the entry; both work once it is collected
    want = _outs([srv.execute(prog, a, enc)], d)
    pend = srv.execute_batch_async(prog, [(a, ref)], 0)
    refused(lambda: srv.release(h), "not been collected")
    refused(lambda: srv.remove_keys(a), "not been collected")
    _same(_outs(srv.execute_batch_result(pend), d), want, "after refusals")
    # a removed tenant's entries go with its keys: its id given to another client names none of them
    srv.remove_keys(a)
    assert srv.bank_info()["stored"] == 0
    assert srv.add_keys(other) == a
    refused(lambda: srv.execute(prog, a, ref), "handle %d" % h, "no such entry")
    h2 = srv.store(a, other.encrypt(client_inputs(d, 4), sig))["image"]
    assert h2 > hl > h
    # no store at all
    plainsrv = b200.B200Server(params, capacity=1)
    plainsrv.add_keys(pub)
    plainsrv.execute(prog, 0, enc)
    with pytest.raises(ValueError, match="store_entries"):
        plainsrv.store(0, enc)
    with pytest.raises(ValueError, match="store_entries"):
        plainsrv.release(1)
    before = plainsrv.launch_count()
    with pytest.raises(ValueError, match="no ciphertext store"):
        plainsrv.execute(prog, 0, ref)
    assert plainsrv.launch_count() == before
    with pytest.raises(ValueError, match="no ciphertext store"):
        pub.execute(prog, ref)
    with pytest.raises(ValueError, match="stored"):
        sec.decrypt(ref, sig)
    info = plainsrv.bank_info()
    assert info["store_entries"] == 0 and info["stored"] == 0 and info["store_bytes"] == 0
    with pytest.raises(ValueError, match="store_entries"):
        b200.B200Server(params, capacity=1, store_entries=-1)


def test_mixed_valuation_through_a_file(tmp_path):
    """a full, a seeded and a stored input cross a file (payload kinds CIPHERTEXT, 18 and 19) and run as before"""
    from eva_b200 import b200, load, save
    d, prog, params, sig, pub, sec = _ctx("feat_bin_mul_11")
    srv = b200.B200Server(params, capacity=1, store_entries=1)
    t = srv.add_keys(pub)
    full, seeded = pub.encrypt(client_inputs(d, 1), sig), sec.encrypt(client_inputs(d, 1), sig)
    one = b200.B200Valuation()
    copy_value(full, one, "b")
    h = srv.store(t, one)["b"]
    x = b200.B200Valuation()
    copy_value(full, x, "a")
    copy_value(seeded, x, "b")
    x.set_stored("c", h)
    save(x, str(tmp_path / "mixed.sealvals"))
    back = load(str(tmp_path / "mixed.sealvals"))
    assert back.get("c") == ("stored", h, None) and back.get("b")[0] == "seeded_cipher" and back.get("a")[0] == "cipher"
    assert np.array_equal(back.get("a")[1], full.get("a")[1]) and back.get_seed("b") == seeded.get_seed("b")
    # a request file: a seeded inline a and the stored b
    save(request(seeded, {"b": h}), str(tmp_path / "req.sealvals"))
    inline = b200.B200Valuation()
    copy_value(seeded, inline, "a")
    copy_value(full, inline, "b")
    _same(_outs([srv.execute(prog, t, load(str(tmp_path / "req.sealvals")))], d), _outs([srv.execute(prog, t, inline)], d), "through a file")


# ------------------------------------------------------------------------------------------------------------ record matching
def record_match(vec_size=4096):
    from eva_b200 import EvaProgram, Input, Output
    from eva_b200.ckks import CKKSCompiler
    from eva_b200.std.numeric import horizontal_sum
    prog = EvaProgram("record_match", vec_size)
    with prog:
        Output("score", horizontal_sum(Input("query") * Input("record")))
    prog.set_output_ranges(30)
    prog.set_input_scales(30)
    return CKKSCompiler().compile(prog)


def test_record_match_meets_the_reference_criterion():
    from eva_b200 import b200, evaluate
    prog, params, sig = record_match()
    pub, sec = b200.generate_keys(params, seed=3)
    srv = b200.B200Server(params, capacity=1, store_entries=1)
    t = srv.add_keys(pub)
    rng = np.random.default_rng(9)
    record = list(rng.uniform(0, 0.1, sig.vec_size))
    h = srv.store(t, sec.encrypt({"record": record}, sig))
    for i in range(3):
        query = list(rng.uniform(0, 0.1, sig.vec_size))
        req = request(pub.encrypt({"query": query}, sig), h)
        got = np.array(sec.decrypt(srv.execute(prog, t, req), sig)["score"])
        want = np.array(evaluate(prog, {"query": query, "record": record})["score"])
        assert np.mean((got - want) ** 2) < 0.01, i
