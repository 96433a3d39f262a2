"""Ciphertext stores larger than the device (max_stored > store_entries) and seeded stores (store_storage="seeded") on the GPU:
every request that names stored entries gives the output bytes of the same request on an un-paged "expanded" store and of the
same ciphertexts sent inline, while entries are evicted and filled under it; the fill and eviction counts are the CPU replay's
(RegionCache::assignAll, test_store_paging.py); and every new error names its option and issues no launch."""
import numpy as np
import pytest

from eva_b200 import program_io as gl
from oracle import oracle as o
from oracle_exec import OracleProgram
from test_compressed_keys_gpu import _same
from test_seeded_inputs_gpu import _ctx, _outs, client_inputs
from test_store_paging import cycling_batches, store_replay
from test_stored_inputs_gpu import copy_value, record_match, request

pytestmark = pytest.mark.gpu

LAYOUTS = [("expanded", "full"), ("expanded", "seeded"), ("seeded", "seeded")]   # (store_storage, ciphertexts stored)


def _encrypt(pub, sec, kind, inputs, sig):
    return (sec.encrypt if kind == "seeded" else pub.encrypt)(inputs, sig)


def _layout_bytes(params, storage, ell, seeded):
    from eva_b200 import _eva_b200 as native
    return native._store_bytes(len(params.prime_bits), params.poly_modulus_degree, storage, ell, seeded)


# ---------------------------------------------------------------------------------------------------- Sobel, every batch evicts
@pytest.mark.parametrize("storage,kind", LAYOUTS)
def test_sobel_cycling_over_four_times_the_entries(storage, kind):
    """store_entries=4, max_stored=64, 16 stored images named 4 at a time (each twice per batch): sync, then async with two slots in
    flight (the second batch's fills wait for the first's gathers).  Equal to an un-paged expanded store and to inline"""
    from eva_b200 import b200
    d, prog, params, sig, pub, sec = _ctx("sobel")
    S = 16
    encs = [_encrypt(pub, sec, kind, client_inputs(d, i), sig) for i in range(S)]
    srv = b200.B200Server(params, capacity=1, store_entries=4, max_stored=64, store_storage=storage)
    ref = b200.B200Server(params, capacity=1, store_entries=S)
    t, rt = srv.add_keys(pub), ref.add_keys(pub)
    want = _outs(ref.execute_batch(prog, [(rt, e) for e in encs]), d)
    before = srv.launch_count()
    handles = [srv.store(t, e)["image"] for e in encs]
    assert srv.launch_count() == before                       # host memory only
    ref_handles = [ref.store(rt, e)["image"] for e in encs]
    ell = len(params.prime_bits) - 1 - d["signature"]["image"]["level"]
    entry, host = _layout_bytes(params, storage, ell, kind == "seeded")
    info = srv.bank_info()
    assert (info["store_entries"], info["max_stored"], info["store_storage"], info["stored"]) == (4, 64, storage, S)
    assert info["store_entry_bytes"] == entry and info["store_bytes"] == 4 * entry and info["store_host_bytes"] == S * host
    assert info["store_resident"] == [] and info["store_fills"] == 0
    assert ref.bank_info()["store_host_bytes"] == 0 and ref.bank_info()["max_stored"] == S
    batches = cycling_batches(S, 4, 8)
    resolved = []

    def reqs(batch, hs):
        return [(t, request(encs[i - 1], {"image": hs[i - 1]})) for i in batch]

    def expect(batch):
        return [want[i - 1] for i in batch]
    for batch in batches:
        _same(_outs(srv.execute_batch(prog, reqs(batch, handles)), d), expect(batch), (storage, kind, "sync", batch))
        _same(_outs(ref.execute_batch(prog, [(rt, r) for _, r in reqs(batch, ref_handles)]), d), expect(batch), "un-paged")
        resolved.append([handles[i - 1] for i in batch])
    for a, b in zip(batches[::2], batches[1::2]):
        ha = srv.execute_batch_async(prog, reqs(a, handles), 0)
        hb = srv.execute_batch_async(prog, reqs(b, handles), 1)
        resolved += [[handles[i - 1] for i in a], [handles[i - 1] for i in b]]
        _same(_outs(srv.execute_batch_result(ha), d), expect(a), (storage, kind, "async first", a))
        _same(_outs(srv.execute_batch_result(hb), d), expect(b), (storage, kind, "async second", b))
    srv.set_options(fuse=8)                                   # one chunk: one gather (and one draw) for all eight references
    _same(_outs(srv.execute_batch(prog, reqs(batches[0], handles)), d), expect(batches[0]), (storage, kind, "fused"))
    resolved.append([handles[i - 1] for i in batches[0]])
    info = srv.bank_info()
    fills, evictions = store_replay(4, resolved)
    assert (info["store_fills"], info["store_evictions"]) == (fills, evictions) and evictions > 0
    assert len(info["store_resident"]) == 4 and set(info["store_resident"]) == {handles[i - 1] for i in batches[0]}


def test_full_and_seeded_entries_in_one_expanded_store():
    """an expanded paged store holds full and seeded ciphertexts side by side; the seeded ones travel as c0 + seed to the host store"""
    from eva_b200 import b200
    d, prog, params, sig, pub, sec = _ctx("sobel")
    encs = [(pub if i % 2 else sec).encrypt(client_inputs(d, 50 + i), sig) for i in range(6)]
    srv = b200.B200Server(params, capacity=1, store_entries=2, max_stored=6)
    t = srv.add_keys(pub)
    want = _outs(srv.execute_batch(prog, [(t, e) for e in encs]), d)
    hs = [srv.store(t, e)["image"] for e in encs]
    ell = len(params.prime_bits) - 1 - d["signature"]["image"]["level"]
    full, seeded = _layout_bytes(params, "expanded", ell, False)[1], _layout_bytes(params, "expanded", ell, True)[1]
    assert srv.bank_info()["store_host_bytes"] == 3 * full + 3 * seeded
    order = [0, 1, 2, 3, 4, 5, 5, 0, 3, 2]
    for i in range(0, len(order), 2):
        pair = order[i:i + 2]
        got = srv.execute_batch(prog, [(t, request(encs[j], {"image": hs[j]})) for j in pair])
        _same(_outs(got, d), [want[j] for j in pair], ("mixed", pair))


# ------------------------------------------------------------------------------------------------------ other programs
def test_record_match_one_stored_one_inline():
    from eva_b200 import b200
    prog, params, sig = record_match()
    pub, sec = b200.generate_keys(params, seed=3)
    srv = b200.B200Server(params, capacity=1, store_entries=1, max_stored=4, store_storage="seeded")
    t = srv.add_keys(pub)
    rng = np.random.default_rng(9)
    records = [sec.encrypt({"record": list(rng.uniform(0, 0.1, sig.vec_size))}, sig) for _ in range(4)]
    handles = [srv.store(t, r) for r in records]
    queries = [pub.encrypt({"query": list(rng.uniform(0, 0.1, sig.vec_size))}, sig) for _ in range(4)]
    for i in (0, 1, 2, 3, 1, 1, 0):
        inline = b200.B200Valuation()
        copy_value(queries[i], inline, "query")
        copy_value(records[i], inline, "record")
        want = srv.execute(prog, t, inline).get("score")
        got = srv.execute(prog, t, request(queries[i], handles[i])).get("score")
        assert got[0] == want[0] == "cipher" and np.array_equal(got[1], want[1]) and got[2] == want[2], i
    assert srv.bank_info()["store_evictions"] >= 4


def test_slot_packed_program():
    from eva_b200 import b200
    from eva_b200.ckks import pack_inputs, pack_program
    d = gl.load_json("sobel")
    prog, params, sig, _ = gl.build_program(d)
    packed, pparams, psig = pack_program(prog, params, sig, 2)
    pub, sec = b200.generate_keys(pparams, seed=12)
    srv = b200.B200Server(pparams, capacity=1, store_entries=2, max_stored=3, store_storage="seeded")
    t = srv.add_keys(pub)
    rng = np.random.default_rng(5)
    encs = [sec.encrypt(pack_inputs([{"image": rng.uniform(0, 0.2, sig.vec_size)} for _ in range(2)], sig, 2), psig) for _ in range(3)]
    want = _outs(srv.execute_batch(packed, [(t, e) for e in encs]), d)
    hs = [srv.store(t, e) for e in encs]
    for pair in ([0, 1], [2, 0], [1, 2], [0, 0]):
        got = srv.execute_batch(packed, [(t, request(encs[i], hs[i])) for i in pair])
        _same(_outs(got, d), [want[i] for i in pair], ("packed k = 2", pair))


def test_key_paging_seeded_keys_and_c1_cache():
    """tenant paging with seeded keys and a c1 cache, and a paged seeded store, all moving at once"""
    from eva_b200 import b200
    d, prog, params, sig, _, _ = _ctx("sobel")
    ctxs = [b200.generate_keys(params, seed=30 + t) for t in range(3)]
    srv = b200.B200Server(params, capacity=2, max_tenants=3, hoist_constants="inline", key_storage="seeded", c1_cache=1,
                          store_entries=2, max_stored=6, store_storage="seeded")
    ref = b200.B200Server(params, capacity=3)
    for p, _ in ctxs:
        srv.add_keys(p)
        ref.add_keys(p)
    encs = {(t, j): ctxs[t][1].encrypt(client_inputs(d, 60 + 2 * t + j), sig) for t in range(3) for j in range(2)}
    hs = {key: srv.store(key[0], e) for key, e in encs.items()}
    for order in ([(0, 0), (1, 0), (0, 0)], [(2, 1), (2, 0)], [(1, 1), (0, 1), (1, 1)], [(2, 0), (0, 0)], [(1, 0)]):
        got = srv.execute_batch(prog, [(t, request(encs[(t, j)], hs[(t, j)])) for t, j in order])
        _same(_outs(got, d), _outs(ref.execute_batch(prog, [(t, encs[(t, j)]) for t, j in order]), d), ("keys, c1 and store paging", order))
    info = srv.bank_info()
    assert info["evictions"] > 0 and info["store_evictions"] > 0 and info["c1_fills"] > 0


def test_zero_digit_redo_refills_its_evicted_entry():
    """the zero-digit ciphertext, stored in a one-entry paged store; a second batch evicts it before the first is collected, and
    collect's redo fills it again and returns the oracle's bits"""
    from eva_b200 import b200
    d = gl.load_json("sobel")
    prog, params, sig, terms = gl.build_program(d)
    orc = o.Oracle(d["poly_modulus_degree"], d["prime_bits"]).keygen(1)
    op = OracleProgram(d, orc)
    op.prepare_keys()
    srv = b200.B200Server(params, capacity=1, store_entries=1, max_stored=2)
    assert list(srv.primes()) == list(orc.primes)
    gks = {int(e): k for e, k in op.gks.items()}
    for e in srv.bank_info()["galois_elements"]:
        gks.setdefault(int(e), orc.galois_key(int(e)))
    t = srv.add_raw_keys(op.rk, gks)
    rng = np.random.default_rng(4)
    (name_, info), = d["signature"].items()
    ell = orc.k - 1 - info["level"]
    scale = 2.0 ** info["scale"]
    vals, V = [], []
    for i in range(2):
        ct = orc.encrypt(orc.encode(rng.uniform(0, 1, d["vec_size"]), scale, ell), seed=3 + i)
        if i == 0:
            c1 = np.stack([orc.ntt_inv(ct[1, r], r) for r in range(ell)])
            c1[1, 7] = 0                                  # one zero coefficient in digit 1
            ct[1] = np.stack([orc.ntt_fwd(c1[r], r) for r in range(ell)])
        v = b200.B200Valuation()
        v.set_cipher(name_, ct, scale)
        vals.append(v)
        V.append(op.run({name_: ("cipher", ct, scale)}))
    reqs = [request(v, srv.store(t, v)) for v in vals]
    built = srv.plans_built()
    ha = srv.execute_batch_async(prog, [(t, reqs[0])], 0)
    hb = srv.execute_batch_async(prog, [(t, reqs[1])], 1)       # evicts the entry batch 0 names
    assert srv.bank_info()["store_resident"] == [reqs[1].get(name_)[1]]
    out_a = srv.execute_batch_result(ha)[0]
    assert srv.plans_built() > built                             # the redo's plans, without the shared mod-up
    info = srv.bank_info()
    assert info["store_resident"] == [reqs[0].get(name_)[1]] and (info["store_fills"], info["store_evictions"]) == (3, 2)
    out_b = srv.execute_batch_result(hb)[0]
    for oname, oid in d["outputs"].items():
        assert np.array_equal(out_a.get(oname)[1], V[0][oid][1])
        assert np.array_equal(out_b.get(oname)[1], V[1][oid][1])


# ------------------------------------------------------------------------------------------------------------------- errors
def test_errors_name_their_option_and_issue_no_launch():
    from eva_b200 import b200
    d, prog, params, sig, pub, sec = _ctx("sobel")
    with pytest.raises(ValueError, match="max_stored"):
        b200.B200Server(params, capacity=1, store_entries=4, max_stored=3)
    with pytest.raises(ValueError, match="max_stored"):
        b200.B200Server(params, capacity=1, max_stored=4)
    with pytest.raises(ValueError, match="store_storage.*compressed"):
        b200.B200Server(params, capacity=1, store_entries=1, store_storage="compressed")
    srv = b200.B200Server(params, capacity=1, store_entries=2, max_stored=4, store_storage="seeded")
    t = srv.add_keys(pub)
    seeded = [sec.encrypt(client_inputs(d, 70 + i), sig) for i in range(5)]
    full = pub.encrypt(client_inputs(d, 80), sig)
    srv.execute_batch(prog, [(t, seeded[0]), (t, seeded[1])])    # plans built and keys resident: what follows counts launches only
    srv.execute(prog, t, seeded[0])

    def refused(fn, *words):
        before, info = srv.launch_count(), srv.bank_info()
        with pytest.raises(ValueError) as e:
            fn()
        for w in words:
            assert w in str(e.value), (w, str(e.value))
        assert srv.launch_count() == before
        after = srv.bank_info()
        assert [after[k] for k in ("stored", "store_fills", "store_resident")] == [info[k] for k in ("stored", "store_fills", "store_resident")]
    refused(lambda: srv.store(t, full), "value image", "full ciphertext", 'store_storage="seeded"')
    hs = [srv.store(t, seeded[i])["image"] for i in range(4)]
    refused(lambda: srv.store(t, seeded[4]), "max_stored=4")
    refs = [request(seeded[i], {"image": hs[i]}) for i in range(4)]
    refused(lambda: srv.execute_batch(prog, [(t, r) for r in refs[:3]]), "3 distinct stored ciphertexts", "store_entries=2")
    refused(lambda: srv.execute_batch(prog, [(t, refs[0]), (t, seeded[2]), (t, refs[1]), (t, refs[2])]), "store_entries=2")
    # release and remove_keys of an entry an uncollected batch names are refused; a released entry's device copy is dropped, and a
    # new ciphertext in its host entry takes a new handle and its own bytes
    want = _outs(srv.execute_batch(prog, [(t, seeded[0]), (t, seeded[4])]), d)
    pend = srv.execute_batch_async(prog, [(t, refs[0]), (t, refs[1])], 0)
    with pytest.raises(RuntimeError, match="not been collected"):
        srv.release(hs[0])
    with pytest.raises(RuntimeError, match="not been collected"):
        srv.remove_keys(t)
    srv.execute_batch_result(pend)
    srv.release(hs[0])
    assert hs[0] not in srv.bank_info()["store_resident"]
    before = srv.launch_count()
    h4 = srv.store(t, seeded[4])["image"]
    assert srv.launch_count() == before and h4 > max(hs)
    got = srv.execute_batch(prog, [(t, refs[1]), (t, request(seeded[4], {"image": h4}))])
    _same(_outs(got, d)[1:], want[1:], "a new entry in a released host entry")
    gone = request(seeded[0], {"image": hs[0]})
    refused(lambda: srv.execute(prog, t, gone), "handle %d" % hs[0], "no such entry")
