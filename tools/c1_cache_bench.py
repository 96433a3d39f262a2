"""Cached c1 rows on one GPU: B200Server(hoist_constants="inline") with key_storage="expanded", key_storage="seeded" and key_storage=
"seeded" with c1_cache (regions holding the expanded c1 rows of the tenants used most), modes alternating within each run (--runs),
outputs compared byte for byte in every call.  Every tenant is added compressed (c0 rows and 32-byte seeds).

  resident     Sobel / Harris, program keys: 32 resident tenants, all cached (c1_cache = 32), 32 instances per step (fuse 1):
               device-resident ops/s (inputs staged once, one replica per instance on its own stream, CUDA events around every step,
               L2 flushed between steps), end-to-end ops/s (two steps in flight) and batch-1 latency
  budget       the same key-bank byte budget (--budget-gb) for every mode: expanded slots, seeded slots, and seeded slots for all 48
               tenants plus as many c1 regions as the rest of the budget holds.  32 instances per step under Zipf-skewed traffic from a
               fixed seed, and under a rotation of 48 tenants, 32 distinct per step (the thrashing case): end-to-end ops/s, fills and
               c1 fills per step
  fill         device time of one evab_expand_seeded_c1 call for one tenant's keys (CUDA events, 50 calls)

The GPU name, power limit and max SM clock are read in the same call.

  python tools/c1_cache_bench.py --workloads sobel harris --runs 2 --steps 20 --out DIR/c1_cache.json
"""
import argparse
import ctypes as C
import gc
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from tenant_paging_bench import compressed, gpu_info, keys_for, measure, uniform  # noqa: E402

B, KEYSETS, BUDGET_TENANTS, ZIPF_S = 32, 8, 48, 1.1
MODES = ("expanded", "seeded", "cached")


def outputs_equal(outs_a, outs_b, names):
    return all(np.array_equal(x.get(n)[1], y.get(n)[1]) for x, y in zip(outs_a, outs_b) for n in names)


def make(b200, params, mode, capacity, c1=0, **kw):
    ks = "expanded" if mode == "expanded" else "seeded"
    return b200.B200Server(params, capacity=capacity, hoist_constants="inline", key_storage=ks, c1_cache=c1 if mode == "cached" else 0, **kw)


def fill_ms(b200, N, primes, nkeys, reps=50):
    """one tenant's c1 expansion: nkeys seeded images of random words (the draw's cost does not depend on them)"""
    import torch
    from eva_b200 import cabi
    lib = cabi.load()
    k = len(primes)
    pa = (C.c_uint64 * k)(*primes)
    ctx = C.c_void_p()
    assert lib.evab_ctx_create(N, pa, k, torch.cuda.current_device(), C.byref(ctx)) == 0, lib.evab_last_error()
    sw = lib.evab_seeded_key_bytes(ctx) // 8
    img = torch.randint(0, 2 ** 62, (nkeys * sw,), dtype=torch.int64, device="cuda")
    rows = torch.zeros_like(img)
    st = torch.cuda.current_stream()
    call = lambda: lib.evab_expand_seeded_c1(ctx, nkeys, img.data_ptr(), rows.data_ptr(), st.cuda_stream)
    for _ in range(5):
        assert call() == 0, lib.evab_last_error()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    for _ in range(reps):
        call()
    b.record(st)
    torch.cuda.synchronize()
    lib.evab_ctx_destroy(ctx)
    return round(a.elapsed_time(b) / reps, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["sobel", "harris"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--budget-gb", type=float, default=1.8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from eva_b200 import b200, program_io
    opts = dict(num_streams=8, fuse=1)
    main_stream = torch.cuda.current_stream()
    streams = [torch.cuda.Stream() for _ in range(B)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def resident(run, steps):
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for i in range(steps):
            flush.zero_()
            ev[i][0].record(main_stream)
            fork = torch.cuda.Event()
            fork.record(main_stream)
            for g in range(B):
                streams[g].wait_event(fork)
                run(i, g, streams[g].cuda_stream)
                e = torch.cuda.Event()
                e.record(streams[g])
                main_stream.wait_event(e)
            ev[i][1].record(main_stream)
        torch.cuda.synchronize()
        return float(np.median([a.elapsed_time(b) for a, b in ev])) * 1e-3

    result = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0), "instances": B, "steps": args.steps, "options": opts,
              "workloads": {}}
    print(result["gpu"], flush=True)
    for wl in args.workloads:
        d = program_io.load_json(os.path.join(ROOT, "workloads", wl + ".json"))
        N = d["poly_modulus_degree"]
        _, params, _, _ = program_io.build_program(d)
        primes = b200.create_coeff_modulus(N, d["prime_bits"])
        rng = np.random.default_rng(7)
        vals = []
        for i in range(B):
            v = b200.B200Valuation()
            for name, info in d["signature"].items():
                v.set_cipher(name, uniform(rng, primes, (2,), len(primes) - 1 - info["level"], N), 2.0 ** info["scale"])
            vals.append(v)
        wout = {}
        # ---- 1. every tenant resident and cached
        prog = program_io.build_program(d)[0]
        srv = {m: make(b200, params, m, B, c1=B) for m in MODES}
        elts = srv["expanded"].bank_info()["galois_elements"]
        keysets = [keys_for(elts, primes, N, 100 + s) for s in range(KEYSETS)]
        comp = [compressed(k, 1100 + i) for i, k in enumerate(keysets)]
        for s in srv.values():
            for t in range(B):
                s.add_compressed_keys(*comp[t % KEYSETS])
            s.set_options(**opts)
        pub = b200.context_from_raw_keys(N, primes, *keysets[0])
        nops = pub.cipher_op_count(prog)
        del pub
        reqs = list(zip(range(B), vals))
        outs = {m: s.execute_batch(prog, reqs) for m, s in srv.items()}
        equal = all(outputs_equal(outs["expanded"], outs[m], d["outputs"]) for m in MODES)
        s0 = main_stream.cuda_stream
        for s in srv.values():
            for r in range(2 * B):
                s.stage_inputs(prog, [(r % B, vals[r % B])], s0, r)
        torch.cuda.synchronize()

        def res(m, steps):
            s = srv[m]
            return resident(lambda i, g, st: s.run_resident(prog, st, 1, g + B * (i % 2), [g]), steps)

        def e2e(m, steps):
            s = srv[m]
            return measure(lambda i: s.execute_batch_async(prog, reqs, i & 1), s.execute_batch_result, steps)

        def lat(m, reps):
            s, ts = srv[m], []
            for r in range(reps):
                t0 = time.perf_counter()
                s.execute(prog, r % B, vals[r % B])
                ts.append(time.perf_counter() - t0)
            return float(np.median(ts))
        for m in srv:
            e2e(m, 2 * args.warmup); res(m, args.warmup); lat(m, args.warmup)
        rate = {"resident": {m: [] for m in srv}, "e2e": {m: [] for m in srv}, "latency_ms": {m: [] for m in srv}}
        for r in range(args.runs):
            for m in (MODES if r % 2 == 0 else MODES[::-1]):
                rate["resident"][m].append(round(B * nops / res(m, args.steps)))
                rate["e2e"][m].append(round(B * nops * args.steps / e2e(m, args.steps)))
                rate["latency_ms"][m].append(round(lat(m, args.steps) * 1e3, 3))
        info = {m: {k: s.bank_info()[k] for k in ("tenant_bytes", "bank_bytes", "c1_cache_bytes", "c1_fills")} for m, s in srv.items()}
        wout["resident"] = {"outputs_equal": equal, "ops_per_s": rate, "bank": info, "cipher_ops_per_instance": nops}
        print(wl, "resident", json.dumps(wout["resident"]), flush=True)
        nkeys = 1 + len(elts)
        del srv, prog, s
        gc.collect()
        # ---- 2. equal bank budget, 48 tenants, 32 instances per step
        budget = int(args.budget_gb * 1e9)
        tb = {m: make(b200, params, m, 1).bank_info()["tenant_bytes"] for m in ("expanded", "seeded")}
        fit = {m: budget // tb[m] for m in tb}
        slots = {"expanded": min(BUDGET_TENANTS, fit["expanded"]), "seeded": min(BUDGET_TENANTS, fit["seeded"])}
        slots["cached"] = slots["seeded"]
        c1 = min(slots["seeded"], fit["seeded"] - slots["seeded"])
        traffic = {
            "zipf": [[int(t) for t in np.minimum(np.random.default_rng(1000 + i).zipf(ZIPF_S, B) - 1, BUDGET_TENANTS - 1)] for i in range(4 * args.steps)],
            "rotation": [[(16 * i + g) % BUDGET_TENANTS for g in range(B)] for i in range(4 * args.steps)],
        }
        prog = program_io.build_program(d)[0]
        srv = {}
        for m in MODES:
            srv[m] = make(b200, params, m, slots[m], c1=c1, max_tenants=BUDGET_TENANTS + 1)
            for t in range(BUDGET_TENANTS):
                srv[m].add_compressed_keys(*comp[t % KEYSETS])
            srv[m].set_options(**opts)
        bout = {"budget_bytes": budget, "slots": slots, "c1_cache": c1, "tenants": BUDGET_TENANTS, "zipf_s": ZIPF_S,
                "bank_bytes": {m: s.bank_info()["bank_bytes"] + s.bank_info()["c1_cache_bytes"] for m, s in srv.items()}}
        for tname, seq in traffic.items():
            batch = lambda i: [(t, vals[g]) for g, t in enumerate(seq[i % len(seq)])]
            o = {m: s.execute_batch(prog, batch(0)) for m, s in srv.items()}
            eq = all(outputs_equal(o["expanded"], o[m], d["outputs"]) for m in MODES)
            for m, s in srv.items():
                measure(lambda i: s.execute_batch_async(prog, batch(i), i & 1), s.execute_batch_result, 2 * args.warmup)
            brate, fills, c1f = ({m: [] for m in srv} for _ in range(3))
            for r in range(args.runs):
                for m in (MODES if r % 2 == 0 else MODES[::-1]):
                    s = srv[m]
                    f0, g0 = s.bank_info()["fills"], s.bank_info()["c1_fills"]
                    dt = measure(lambda i: s.execute_batch_async(prog, batch(i), i & 1), s.execute_batch_result, args.steps)
                    brate[m].append(round(B * nops * args.steps / dt))
                    fills[m].append((s.bank_info()["fills"] - f0) / args.steps)
                    c1f[m].append((s.bank_info()["c1_fills"] - g0) / args.steps)
            bout[tname] = {"outputs_equal": eq, "e2e_ops_per_s": brate, "fills_per_step": fills, "c1_fills_per_step": c1f,
                           "distinct_per_step": float(np.mean([len(set(b)) for b in seq]))}
        wout["equal_budget"] = bout
        print(wl, "equal_budget", json.dumps(bout), flush=True)
        del srv, prog, s
        gc.collect()
        # ---- 3. one fill
        wout["fill_ms"] = fill_ms(b200, N, primes, nkeys)
        wout["fill_keys"] = nkeys
        print(wl, "fill_ms", wout["fill_ms"], flush=True)
        result["workloads"][wl] = wout
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
