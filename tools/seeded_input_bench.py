"""Seed-compressed input ciphertexts on one GPU: what sending c0 + a 32-byte seed instead of (c0, c1) does to time.

A compiled workload (Sobel, Harris) runs with 32 instances per step (fuse 1, 8 streams), end to end with two steps in flight
(execute_batch_async / execute_batch_result, as bench.py measures), under two arms that alternate within each run (--runs):

  full      the valuations hold full ciphertexts (set_cipher): c0 and c1, 2 ell N words each
  seeded    the same ciphertexts as B200Secret.encrypt makes them (c0, ell N words, and a seed): c1 is expanded on the device
            while the inputs are staged

The full ciphertexts are the seeded ones with c1 replayed on the host by the numpy restatement of the rule
(tests/test_seeded_inputs.py), so both arms carry the same ciphertexts and their outputs must be byte-equal (checked).  Both arms
also run on a B200Server with 32 resident tenants.

Also measured, with CUDA events on one stream: one 32-instance chunk's staging split into the c0 uploads (page-locked host ->
device, one per instance as the executor stages), the one expansion launch of the chunk (evab_expand_cipher_uniform), and for
comparison the full-ciphertext uploads; the expansion kernel alone, averaged over many launches; and B200Public.stage_inputs of a
fused 32-instance chunk in both arms.  H2D bytes per step are counted from shapes; the GPU name and power limit are read in the
same run.

  python tools/seeded_input_bench.py --workloads sobel harris --runs 2 --steps 20 --out DIR/seeded.json
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

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


def full_of(val, N, primes):
    from eva_b200 import b200
    from test_seeded_inputs import np_cipher_c1
    out = b200.B200Valuation()
    for n in val.names():
        kind, arr, scale = val.get(n)
        if kind == "seeded_cipher":
            c1, _ = np_cipher_c1(val.get_seed(n), N, primes, arr.shape[0])
            out.set_cipher(n, np.ascontiguousarray(np.stack([arr, c1])), scale)
        elif kind == "plain":
            out.set_plain(n, arr, scale)
        else:
            out.set_raw(n, list(arr))
    return out


def staging_costs(N, primes, ell, reps=20, launches=200):
    """event-timed (ms) on one stream: the c0 uploads of a 32-instance chunk, its expansion launch, the full-ciphertext uploads"""
    import torch
    from eva_b200 import cabi
    lib = cabi.load()
    k = len(primes)
    pa = np.array(primes, dtype=np.uint64)
    h = C.c_void_p()
    assert lib.evab_ctx_create(C.c_uint64(N), pa.ctypes.data_as(C.POINTER(C.c_uint64)), k, 0, C.byref(h)) == 0
    P = ell * N
    rng = np.random.default_rng(5)
    c0 = torch.from_numpy(rng.integers(0, 1 << 59, B * P, dtype=np.int64)).pin_memory()
    full = torch.from_numpy(rng.integers(0, 1 << 59, 2 * B * P, dtype=np.int64)).pin_memory()
    dev = torch.empty(2 * B * P, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream()
    sp = C.c_void_p(st.cuda_stream)
    seeds = C.c_char_p(rng.integers(0, 256, 32 * B, dtype=np.uint8).tobytes())
    ptrs = (C.c_void_p * B)(*[dev.data_ptr() + 8 * (2 * b + 1) * P for b in range(B)])
    ells = (C.c_int * B)(*([ell] * B))

    def up_c0():
        for b in range(B):
            assert lib.evab_upload(h, C.c_void_p(dev.data_ptr() + 16 * b * P), C.c_void_p(c0.data_ptr() + 8 * b * P), 8 * P, sp) == 0

    def expand():
        assert lib.evab_expand_cipher_uniform(h, B, seeds, ptrs, ells, pa.ctypes.data_as(C.POINTER(C.c_uint64)), sp) == 0

    def up_full():
        for b in range(B):
            assert lib.evab_upload(h, C.c_void_p(dev.data_ptr() + 16 * b * P), C.c_void_p(full.data_ptr() + 16 * b * P), 16 * P, sp) == 0

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
    r = {"c0_upload_ms": timed(up_c0), "expand_ms": timed(expand), "full_upload_ms": timed(up_full),
         "expand_alone_ms_per_launch": timed(expand, launches), "launches_averaged": launches,
         "c0_bytes": B * P * 8, "full_bytes": 2 * B * P * 8, "expand_words_written": B * P}

    def seeded_stage():
        up_c0(); expand()
    r["seeded_stage_together_ms"] = timed(seeded_stage)
    torch.cuda.synchronize()
    lib.evab_ctx_destroy(h)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["sobel", "harris"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from eva_b200 import b200, program_io
    opts = dict(num_streams=8, fuse=1)
    result = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0), "instances": B, "steps": args.steps, "options": opts,
              "workloads": {}}
    print(result["gpu"], flush=True)
    for wl in args.workloads:
        d = program_io.load_json(os.path.join(ROOT, "workloads", wl + ".json"))
        N = d["poly_modulus_degree"]
        prog, params, sig, _ = program_io.build_program(d)
        pub, sec = b200.generate_keys(params, seed=11)
        primes = list(pub.primes())
        rng = np.random.default_rng(7)
        seeded = [sec.encrypt({n: list(rng.uniform(0.0, 0.2, d["vec_size"])) for n in d["signature"]}, sig) for _ in range(B)]
        full = [full_of(v, N, primes) for v in seeded]
        srv = b200.B200Server(params, capacity=B)
        tenants = [srv.add_keys(pub) for _ in range(B)]
        pub.set_options(**opts)
        srv.set_options(**opts)
        nops = pub.cipher_op_count(prog)
        arms = {"full": (pub, full), "seeded": (pub, seeded), "server_full": (srv, full), "server_seeded": (srv, seeded)}

        def batch(name):
            ctx, vals = arms[name]
            return vals if ctx is pub else list(zip(tenants, vals))

        def e2e(name, steps):
            ctx = arms[name][0]
            b_ = batch(name)
            return measure(lambda i: ctx.execute_batch_async(prog, b_, i & 1), ctx.execute_batch_result, steps)
        for name in arms:   # plans, replicas, graphs, both submit slots, the page-locked pool
            e2e(name, 2 * max(3, args.warmup))
        # byte-equal outputs at the timed size
        outs = {name: arms[name][0].execute_batch(prog, batch(name)) for name in arms}
        same = all(np.array_equal(outs[a][i].get(n)[1], outs["full"][i].get(n)[1]) for a in arms for i in range(B) for n in d["outputs"])
        rates = {k: [] for k in arms}
        for r in range(args.runs):
            for name in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                rates[name].append(B * nops * args.steps / e2e(name, args.steps))
        # B200Public.stage_inputs of one fused 32-instance chunk (plan replica of batch 32), event-timed
        st = torch.cuda.Stream()
        stage = {}
        pub.set_options(num_streams=8, fuse=B)
        for name in ("full", "seeded", "full", "seeded"):
            vals = arms[name][1]
            pub.stage_inputs(prog, vals, st.cuda_stream, 0)
            ts = []
            for _ in range(10):
                a, b_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(st)
                pub.stage_inputs(prog, vals, st.cuda_stream, 0)
                b_.record(st)
                b_.synchronize()
                ts.append(a.elapsed_time(b_))
            stage.setdefault(name, []).append(float(np.median(ts)))
        pub.set_options(**opts)
        ell = {n: len(primes) - 1 - info["level"] for n, info in d["signature"].items() if info["type"] == "Cipher"}
        out = {
            "cipher_ops_per_instance": nops,
            "e2e_ops_per_s": {k: [round(x) for x in v] for k, v in rates.items()},
            "e2e_ops_per_s_median": {k: round(float(np.median(v))) for k, v in rates.items()},
            "outputs_byte_equal": bool(same),
            "h2d_input_bytes_per_step": {"full": B * sum(2 * e * N * 8 for e in ell.values()), "seeded": B * sum(e * N * 8 for e in ell.values())},
            "stage_inputs_chunk_ms": {k: [round(x, 4) for x in v] for k, v in stage.items()},
            "one_chunk": staging_costs(N, primes, max(ell.values())),
        }
        print(wl, json.dumps(out), flush=True)
        result["workloads"][wl] = out
        del srv, pub, sec
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
