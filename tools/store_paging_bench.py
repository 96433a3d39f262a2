"""Ciphertext stores larger than the device on one GPU: what paging stored ciphertexts from page-locked host memory
(max_stored > store_entries) and keeping seeded entries compressed (store_storage="seeded") cost.

Event-timed on one stream, Sobel's shape (N = 16384, the image at ell = 4):
  fill        one entry written from page-locked host memory, as the store's fill does it: a full ciphertext (one upload of
              2 ell N words), a seeded one into the expanded layout (an upload of c0 and the draw of c1), and a seeded one into
              the seeded layout (an upload of c0 only)
  staging     the stored inputs of a 32-instance chunk: one gather of the whole entries (expanded layout) against one gather of
              the c0 rows and one evab_expand_cipher_uniform call over the 32 seeds (seeded layout)

End to end, Sobel with its image stored, 32 instances per step (fuse 1, 8 streams), two steps in flight
(execute_batch_async / execute_batch_result, as bench.py measures), arms alternating within each run (--runs):
  unpaged            store_entries = 32, every entry on the device (today's store)
  hits / hits_seeded store_entries = 32, max_stored = 64, every step names the same 32 entries (all hits once warm)
  twice / twice_seeded
                     store_entries = 32, max_stored = 64, steps alternate between two sets of 32 entries: every step fills all
                     32 device entries, and each fill waits for the gathers of the step before it
The outputs of every arm are byte-equal to the inline request's (checked).  The GPU name, its power limit and its max SM clock
are read in the same run.

  python tools/store_paging_bench.py --runs 3 --steps 20 --out DIR/store_paging.json
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B = 32


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def measure(submit, collect, steps):
    """seconds for `steps` steps with two in flight (slots 0 and 1)"""
    t0 = time.perf_counter()
    pending = None
    for i in range(steps):
        nxt = submit(i)
        if pending is not None:
            collect(pending)
        pending = nxt
    collect(pending)
    return time.perf_counter() - t0


def sobel():
    from eva_b200 import program_io
    prog, params, sig, _ = program_io.build_program(program_io.load_json(os.path.join(ROOT, "workloads", "sobel.json")))
    return prog, params, sig


def device_costs(N, primes, ell, reps=20, launches=100):
    """event-timed (ms, medians) fills of one entry and staging of one chunk of B entries"""
    import torch
    from eva_b200 import cabi
    lib = cabi.load()
    pa = np.array(primes, dtype=np.uint64)
    h = C.c_void_p()
    assert lib.evab_ctx_create(C.c_uint64(N), pa.ctypes.data_as(C.POINTER(C.c_uint64)), len(primes), 0, C.byref(h)) == 0
    R = ell * N                     # words of one row set (c0 or c1)
    rng = np.random.default_rng(5)
    host = torch.from_numpy(rng.integers(0, 1 << 59, B * 2 * R, dtype=np.int64)).pin_memory()
    store = torch.from_numpy(rng.integers(0, 1 << 59, B * 2 * R, dtype=np.int64)).cuda()
    arena = torch.empty(B * 2 * R, dtype=torch.int64, device="cuda")
    seeds = np.frombuffer(rng.bytes(32 * B), dtype=np.uint8).copy()
    ells = np.full(B, ell, dtype=np.int32)
    st = torch.cuda.current_stream()
    sp = C.c_void_p(st.cuda_stream)
    u64p = C.POINTER(C.c_uint64)

    def upload(dst, words):
        assert lib.evab_upload(h, C.c_void_p(dst), C.c_void_p(host.data_ptr()), 8 * words, sp) == 0

    def draw(c1_ptrs):
        n = len(c1_ptrs)
        assert lib.evab_expand_cipher_uniform(h, n, seeds.ctypes.data_as(C.POINTER(C.c_uint8)), (C.c_void_p * n)(*c1_ptrs),
                                              ells.ctypes.data_as(C.POINTER(C.c_int)), pa.ctypes.data_as(u64p), sp) == 0

    def gather(words):
        src = (C.c_void_p * B)(*[store.data_ptr() + 8 * b * 2 * R for b in range(B)])
        dst = (C.c_void_p * B)(*[arena.data_ptr() + 8 * b * 2 * R for b in range(B)])
        w = np.full(B, words, dtype=np.uint64)
        assert lib.evab_gather_ciphers(h, B, src, dst, w.ctypes.data_as(u64p), sp) == 0

    def timed(fn, n):
        fn()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            for _ in range(n):
                fn()
            b.record(st)
            b.synchronize()
            ts.append(a.elapsed_time(b) / n)
        return float(np.median(ts))
    d0 = store.data_ptr()
    fill = {
        "full_upload_ms": timed(lambda: upload(d0, 2 * R), 20),
        "seeded_into_expanded_ms": timed(lambda: (upload(d0, R), draw([d0 + 8 * R])), 20),
        "seeded_into_seeded_ms": timed(lambda: upload(d0, R), 20),
        "entry_host_bytes": {"full": 2 * R * 8, "seeded": R * 8},
    }
    c1s = [arena.data_ptr() + 8 * (b * 2 * R + R) for b in range(B)]
    staging = {
        "instances": B,
        "expanded_gather_ms": timed(lambda: gather(2 * R), launches),
        "seeded_c0_gather_ms": timed(lambda: gather(R), launches),
        "seeded_draw_ms": timed(lambda: draw(c1s), launches),
        "seeded_gather_plus_draw_ms": timed(lambda: (gather(R), draw(c1s)), launches),
    }
    torch.cuda.synchronize()
    lib.evab_ctx_destroy(h)
    return {"fill_per_entry": fill, "staging_chunk": staging}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from eva_b200 import b200
    opts = dict(num_streams=8, fuse=1)
    prog, params, sig = sobel()
    N = params.poly_modulus_degree
    pub, sec = b200.generate_keys(params, seed=11)
    primes = list(pub.primes())
    ell = len(primes) - 1 - sig.inputs["image"].level
    result = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0), "workload": "sobel", "N": N, "ell": ell,
              "instances": B, "steps": args.steps, "options": opts}
    print(result["gpu"], flush=True)
    result.update(device_costs(N, primes, ell))
    print(json.dumps({k: result[k] for k in ("fill_per_entry", "staging_chunk")}), flush=True)

    rng = np.random.default_rng(7)
    encs = [sec.encrypt({"image": list(rng.uniform(0.0, 0.1, sig.vec_size))}, sig) for _ in range(2 * B)]
    arms, servers = {}, []

    def server(storage, max_stored, sets):
        srv = b200.B200Server(params, capacity=1, store_entries=B, max_stored=max_stored, store_storage=storage)
        t = srv.add_keys(pub)
        srv.set_options(**opts)
        reqs = []
        for e in encs[:B * sets]:
            r = b200.B200Valuation()
            r.set_stored("image", srv.store(t, e)["image"])
            reqs.append((t, r))
        servers.append(srv)
        return srv, [reqs[s * B:(s + 1) * B] for s in range(sets)]
    arms["unpaged"] = server("expanded", None, 1)
    arms["hits"] = server("expanded", 2 * B, 1)
    arms["hits_seeded"] = server("seeded", 2 * B, 1)
    arms["twice"] = server("expanded", 2 * B, 2)
    arms["twice_seeded"] = server("seeded", 2 * B, 2)
    ref = servers[0]
    want = [ref.execute_batch(prog, [(0, e) for e in encs[s * B:(s + 1) * B]]) for s in range(2)]

    def e2e(name, steps):
        srv, sets = arms[name]
        return measure(lambda i: srv.execute_batch_async(prog, sets[i % len(sets)], i & 1), srv.execute_batch_result, steps)
    same = {}
    for name, (srv, sets) in arms.items():
        e2e(name, 2 * max(3, args.warmup))
        same[name] = all(np.array_equal(got.get(n)[1], w.get(n)[1]) for s in range(len(sets))
                         for got, w in zip(srv.execute_batch(prog, sets[s]), want[s]) for n in prog.outputs)
    rates = {k: [] for k in arms}
    for r in range(args.runs):
        for name in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
            rates[name].append(B * args.steps / e2e(name, args.steps))
    result["e2e_requests_per_s"] = {k: [round(x, 1) for x in v] for k, v in rates.items()}
    result["e2e_requests_per_s_median"] = {k: round(float(np.median(v)), 1) for k, v in rates.items()}
    result["outputs_byte_equal"] = same
    result["bank_info"] = {name: {k: srv.bank_info()[k] for k in ("store_entries", "max_stored", "store_storage", "store_bytes",
                                                                   "store_host_bytes", "store_fills", "store_evictions")}
                           for name, (srv, _) in arms.items()}
    print(json.dumps({k: result[k] for k in ("e2e_requests_per_s_median", "outputs_byte_equal")}), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
