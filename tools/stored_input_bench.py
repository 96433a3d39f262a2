"""Server-resident input ciphertexts on one GPU: what naming a stored ciphertext by handle, instead of sending it with every
request, does to request size and time.

A B200Server with 32 tenants (each its own stored data) runs 32 instances per step (fuse 1, 8 streams), end to end with two steps
in flight (execute_batch_async / execute_batch_result, as bench.py measures), under two arms that alternate within each run
(--runs):

  inline    every request carries its ciphertexts in full
  stored    the tenant's data ciphertext is in the server's store (B200Server.store) and the request names it by handle; the
            staging copies it into the arena on the device (evab_gather_ciphers) instead of uploading it

Workloads: record matching, score = horizontal_sum(query * record) (compiled here, vec_size 4096), with `query` fresh per request
and `record` stored; and Sobel (workloads/sobel.json) with the image stored.  Both arms carry the same ciphertexts, so their
outputs must be byte-equal (checked).

Also measured, with CUDA events on one stream: the staging of the stored input for one chunk of 1 and of 32 instances, as
page-locked host -> device uploads (one per instance, as the executor stages an inline ciphertext) against one
evab_gather_ciphers launch (k_gather_words) from a device store.  Request bytes per instance are counted from shapes; the GPU
name and power limit are read in the same run.

  python tools/stored_input_bench.py --runs 2 --steps 20 --out DIR/stored.json
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
HANDLE_BYTES = 8


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


def sobel():
    from eva_b200 import program_io
    prog, params, sig, _ = program_io.build_program(program_io.load_json(os.path.join(ROOT, "workloads", "sobel.json")))
    return prog, params, sig


def staging_costs(N, primes, ell, reps=20, launches=200):
    """event-timed (ms) on one stream: the stored input of a chunk of 1 and of B instances as uploads and as one gather"""
    import torch
    from eva_b200 import cabi
    lib = cabi.load()
    pa = np.array(primes, dtype=np.uint64)
    h = C.c_void_p()
    assert lib.evab_ctx_create(C.c_uint64(N), pa.ctypes.data_as(C.POINTER(C.c_uint64)), len(primes), 0, C.byref(h)) == 0
    W = 2 * ell * N
    rng = np.random.default_rng(5)
    host = torch.from_numpy(rng.integers(0, 1 << 59, B * W, dtype=np.int64)).pin_memory()
    store = torch.from_numpy(rng.integers(0, 1 << 59, B * W, dtype=np.int64)).cuda()
    arena = torch.empty(B * W, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream()
    sp = C.c_void_p(st.cuda_stream)

    def upload(n):
        for b in range(n):
            assert lib.evab_upload(h, C.c_void_p(arena.data_ptr() + 8 * b * W), C.c_void_p(host.data_ptr() + 8 * b * W), 8 * W, sp) == 0

    def gather(n):
        src = (C.c_void_p * n)(*[store.data_ptr() + 8 * b * W for b in range(n)])
        dst = (C.c_void_p * n)(*[arena.data_ptr() + 8 * b * W for b in range(n)])
        words = np.full(n, W, dtype=np.uint64)
        assert lib.evab_gather_ciphers(h, n, src, dst, words.ctypes.data_as(C.POINTER(C.c_uint64)), sp) == 0

    def timed(fn, n=1):
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
    r = {}
    for n in (1, B):
        ms = timed(lambda: gather(n), launches)
        r["chunk_%d" % n] = {"h2d_upload_ms": timed(lambda: upload(n)), "gather_ms": timed(lambda: gather(n)),
                             "gather_ms_per_launch_averaged": ms, "launches_averaged": launches, "bytes": n * W * 8,
                             "gather_device_GBps": round(2 * n * W * 8 / ms / 1e6, 1)}   # read + write
    torch.cuda.synchronize()
    lib.evab_ctx_destroy(h)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["record_match", "sobel"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from eva_b200 import b200
    opts = dict(num_streams=8, fuse=1)
    result = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0), "instances": B, "tenants": B, "steps": args.steps,
              "options": opts, "workloads": {}}
    print(result["gpu"], flush=True)
    for wl in args.workloads:
        prog, params, sig = {"record_match": record_match, "sobel": sobel}[wl]()
        stored_name = {"record_match": "record", "sobel": "image"}[wl]
        N = params.poly_modulus_degree
        pub, _ = b200.generate_keys(params, seed=11)
        primes = list(pub.primes())
        srv = b200.B200Server(params, capacity=B, store_entries=B)
        tenants = [srv.add_keys(pub) for _ in range(B)]
        srv.set_options(**opts)
        rng = np.random.default_rng(7)
        inline, stored = [], []
        for t in tenants:
            enc = pub.encrypt({n: list(rng.uniform(0.0, 0.1, sig.vec_size)) for n in sig.inputs}, sig)
            data = b200.B200Valuation()
            kind, arr, scale = enc.get(stored_name)
            data.set_cipher(stored_name, arr, scale)
            handle = srv.store(t, data)[stored_name]
            req = b200.B200Valuation()
            for n in enc.names():
                if n == stored_name:
                    req.set_stored(n, handle)
                else:
                    req.set_cipher(n, *enc.get(n)[1:])
            inline.append((t, enc))
            stored.append((t, req))
        arms = {"inline": inline, "stored": stored}

        def e2e(name, steps):
            return measure(lambda i: srv.execute_batch_async(prog, arms[name], i & 1), srv.execute_batch_result, steps)
        for name in arms:   # plans, replicas, graphs, both submit slots, the page-locked pool
            e2e(name, 2 * max(3, args.warmup))
        outs = {name: srv.execute_batch(prog, arms[name]) for name in arms}
        same = all(np.array_equal(outs["stored"][i].get(n)[1], outs["inline"][i].get(n)[1]) for i in range(B) for n in prog.outputs)
        rates = {k: [] for k in arms}
        for r in range(args.runs):
            for name in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                rates[name].append(B * args.steps / e2e(name, args.steps))
        ells = {n: len(primes) - 1 - info.level for n, info in sig.inputs.items()}
        cipher_bytes = {n: 2 * e * N * 8 for n, e in ells.items()}
        out = {
            "N": N, "ell": ells, "stored_input": stored_name,
            "request_bytes_per_instance": {"inline": sum(cipher_bytes.values()),
                                           "stored": sum(b for n, b in cipher_bytes.items() if n != stored_name) + HANDLE_BYTES},
            "e2e_requests_per_s": {k: [round(x, 1) for x in v] for k, v in rates.items()},
            "e2e_requests_per_s_median": {k: round(float(np.median(v)), 1) for k, v in rates.items()},
            "outputs_byte_equal": bool(same),
            "store_bytes": srv.bank_info()["store_bytes"],
            "staging": staging_costs(N, primes, ells[stored_name]),
        }
        print(wl, json.dumps(out), flush=True)
        result["workloads"][wl] = out
        del srv, pub
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
