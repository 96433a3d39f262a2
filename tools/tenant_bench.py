"""Multi-tenant serving on one GPU: ops/s of a compiled workload (Sobel, Harris) with 32 instances per step under four key
arrangements, measured as bench.py measures: device-resident (inputs staged once, one plan replica per instance on its own stream,
CUDA events around every step, L2 flushed between steps) and end to end with two steps in flight (execute_batch_async /
execute_batch_result: host valuations in, host valuations out):

  (a) one B200Public, one key set                       (bench.py's shape)
  (b) B200Server, all instances on one tenant           (cost of the per-instance key indirection)
  (c) B200Server, 32 distinct tenants
  (d) 32 B200Public contexts, one instance each         (what a server does without a key bank)

The arms alternate within each run (--runs).  --no-rotation-sums builds every plan without the weighted rotation sums, so that
the rotations run through evab_rotate_modup_many (k_rot_many).  Also reported: device memory each arm takes (free-memory drop over its set-up and warm-up:
keys, bank, plan arenas, pool caching) and the time to the first result of a newly registered tenant in (c) against a newly
created context in (d) (the latter builds a plan, allocates its arena and captures its graph).  Keys and ciphertexts are uniform
residues (valid evaluator inputs), seeded.

  python tools/tenant_bench.py --workloads sobel harris --runs 4 --steps 20 --out DIR/tenants.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def uniform(rng, primes, prefix, nres, N):
    a = np.empty(tuple(prefix) + (nres, N), dtype=np.uint64)
    for j in range(nres):
        a[..., j, :] = rng.integers(0, primes[j], size=tuple(prefix) + (N,), dtype=np.uint64)
    return a


def keys_for(elts, primes, N, seed):
    rng = np.random.default_rng(seed)
    k = len(primes)
    return uniform(rng, primes, (k - 1, 2), k, N), {int(e): uniform(rng, primes, (k - 1, 2), k, N) for e in elts}


def measure(submit, collect, steps):
    """seconds for `steps` steps with two in flight (slots 0 and 1)"""
    t0 = time.perf_counter()
    pending = None
    for i in range(steps):
        nxt = submit(i & 1)
        if pending is not None:
            collect(pending)
        pending = nxt
    collect(pending)
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["sobel", "harris"])
    ap.add_argument("--instances", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--no-rotation-sums", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from eva_b200 import b200, program_io
    B = args.instances
    opts = dict(num_streams=8, rotation_sums=not args.no_rotation_sums)
    main_stream = torch.cuda.current_stream()
    streams = [torch.cuda.Stream() for _ in range(B)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > the 50 MB L2

    def resident(run, steps):
        """median step time (s) of `steps` device-resident steps: run(g, stream) enqueues instance g's plan replica"""
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for i in range(steps):
            flush.zero_()
            ev[i][0].record(main_stream)
            fork = torch.cuda.Event()
            fork.record(main_stream)
            for g in range(B):
                streams[g].wait_event(fork)
                run(g, streams[g].cuda_stream)
                e = torch.cuda.Event()
                e.record(streams[g])
                main_stream.wait_event(e)
            ev[i][1].record(main_stream)
        torch.cuda.synchronize()
        return float(np.median([a.elapsed_time(b) for a, b in ev])) * 1e-3
    result = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0), "instances": B, "steps": args.steps, "options": opts, "workloads": {}}
    print(result["gpu"], flush=True)
    for wl in args.workloads:
        d = program_io.load_json(os.path.join(ROOT, "workloads", wl + ".json"))
        N = d["poly_modulus_degree"]
        prog, params, sig, _ = program_io.build_program(d)
        primes = b200.create_coeff_modulus(N, d["prime_bits"])
        rng = np.random.default_rng(7)
        vals = []
        for i in range(B):
            v = b200.B200Valuation()
            for name, info in d["signature"].items():
                ell = len(primes) - 1 - info["level"]
                v.set_cipher(name, uniform(rng, primes, (2,), ell, N), 2.0 ** info["scale"])
            vals.append(v)
        single = [(0, v) for v in vals]
        multi = [(t, v) for t, v in enumerate(vals)]

        def free():
            torch.cuda.synchronize()
            return torch.cuda.mem_get_info()[0]

        def warm(sub, col):   # plans, replicas, graphs, both slots, the page-locked pool
            measure(sub, col, 2 * max(3, args.warmup))
        # ---- set-up and warm-up of every arm; device memory taken = the free-memory drop over it
        mem = {}
        f0 = free()
        server = b200.B200Server(params, capacity=B + 1)
        elts = server.bank_info()["galois_elements"]
        for t in range(B):
            server.add_raw_keys(*keys_for(elts, primes, N, 100 + t))
        server.set_options(**opts)
        arms = {"b_server_one_tenant": (lambda s: server.execute_batch_async(prog, single, s), server.execute_batch_result),
                "c_server_32_tenants": (lambda s: server.execute_batch_async(prog, multi, s), server.execute_batch_result)}
        for sub, col in arms.values():
            warm(sub, col)
        mem["server_b_c"] = f0 - free()
        f0 = free()
        pub = b200.context_from_raw_keys(N, primes, *keys_for(elts, primes, N, 100))
        pub.set_options(**opts)
        arms["a_one_context"] = (lambda s: pub.execute_batch_async(prog, vals, s), pub.execute_batch_result)
        warm(*arms["a_one_context"])
        mem["one_context_a"] = f0 - free()
        f0 = free()
        pubs = []
        for t in range(B):
            p = b200.context_from_raw_keys(N, primes, *keys_for(elts, primes, N, 100 + t))
            p.set_options(**opts)
            pubs.append(p)
        arms["d_32_contexts"] = (lambda s: [p.execute_batch_async(prog, [v], s) for p, v in zip(pubs, vals)],
                                 lambda hs: [p.execute_batch_result(h) for p, h in zip(pubs, hs)])
        warm(*arms["d_32_contexts"])
        mem["contexts_d"] = f0 - free()
        arms = {k: arms[k] for k in sorted(arms)}
        mem_server = server.bank_info()
        rates = {k: [] for k in arms}
        nops = pub.cipher_op_count(prog)
        # device-resident: instance g on plan replica g (batch 1) of its arm, staged once
        s0 = main_stream.cuda_stream
        for g in range(B):
            pub.stage_inputs(prog, [vals[g]], s0, g)
            pubs[g].stage_inputs(prog, [vals[g]], s0, 0)
        torch.cuda.synchronize()
        on_server = lambda g, st: server.run_resident(prog, st, 1, g)
        res_runs = {"a_one_context": lambda g, st: pub.run_resident(prog, st, 1, g), "b_server_one_tenant": on_server,
                    "c_server_32_tenants": on_server, "d_32_contexts": lambda g, st: pubs[g].run_resident(prog, st, 1, 0)}
        res_rates = {k: [] for k in arms}

        def stage(name):   # (b) and (c) share the server's replicas: their tenants are staged before each measurement
            if name in ("b_server_one_tenant", "c_server_32_tenants"):
                for g in range(B):
                    server.stage_inputs(prog, [(0 if name.startswith("b_") else g, vals[g])], s0, g)
                torch.cuda.synchronize()
        for name in arms:
            stage(name)
            resident(res_runs[name], max(3, args.warmup))
        for r in range(args.runs):
            for name, (sub, col) in (list(arms.items()) if r % 2 == 0 else list(arms.items())[::-1]):
                stage(name)
                res_rates[name].append(B * nops / resident(res_runs[name], args.steps))
                dt = measure(sub, col, args.steps)
                rates[name].append(B * nops * args.steps / dt)
        # ---- time to the first result of a new client: (c) register a tenant and execute; (d) create a context and execute
        t0 = time.perf_counter()
        t_new = server.add_raw_keys(*keys_for(elts, primes, N, 999))
        t_reg = time.perf_counter() - t0
        server.execute(prog, t_new, vals[0])
        t_first_c = time.perf_counter() - t0
        t0 = time.perf_counter()
        p_new = b200.context_from_raw_keys(N, primes, *keys_for(elts, primes, N, 999))
        p_new.set_options(**opts)
        t_ctx = time.perf_counter() - t0
        p_new.execute(prog, vals[0])
        t_first_d = time.perf_counter() - t0
        plan_bytes = pub.plan_stats(prog, 1, 0)["arena_bytes"]
        out = {
            "cipher_ops_per_instance": nops,
            "resident_ops_per_s": {k: [round(x) for x in v] for k, v in res_rates.items()},
            "resident_ops_per_s_median": {k: round(float(np.median(v))) for k, v in res_rates.items()},
            "e2e_ops_per_s": {k: [round(x) for x in v] for k, v in rates.items()},
            "e2e_ops_per_s_median": {k: round(float(np.median(v))) for k, v in rates.items()},
            "bank": {k: mem_server[k] for k in ("capacity", "tenants", "tenant_bytes", "key_bytes_per_tenant", "hoist_const_bytes_per_tenant", "bank_bytes")},
            "arena_bytes_one_instance_plan": plan_bytes,
            "device_bytes_taken": mem,
            "first_result_new_tenant_s": {"register": t_reg, "register_and_execute": t_first_c},
            "first_result_new_context_s": {"create": t_ctx, "create_and_execute": t_first_d},
        }
        print(wl, json.dumps(out), flush=True)
        result["workloads"][wl] = out
        del pubs, pub, server, p_new
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
