"""Seeded key slots on one GPU: B200Server(hoist_constants="inline", key_storage="expanded") against key_storage="seeded" (slots hold
each key's c0 rows and seed, the key-switch inner products draw the uniform half), arms alternating within each run (--runs), outputs
compared byte for byte in every call.  Every tenant is added compressed (c0 rows and 32-byte seeds), the only form a seeded server
takes; the expanded server expands it on the device.

  throughput   Sobel / Harris, program and power-of-two keys: 32 resident tenants, 32 instances per step (fuse 1): device-resident ops/s
               (inputs staged once, one replica per instance on its own stream, CUDA events around every step, L2 flushed between
               steps), end-to-end ops/s (two steps in flight) and batch-1 latency
  kernels      device time per step of k_rot_wsum_ip, k_rot_many and k_ks_inner (torch.profiler, a separate pass)
  budget       the same key-bank byte budget for both modes (--budget-gb): the slots each mode gets, 48 tenants rotated 32 distinct per
               step; the expanded bank pages, the seeded bank holds them all.  Fills per step, and the mean device time of one fill
               (the pager's stream is timed around a step that only fills)

The GPU name, power limit and max SM clock are read in the same call.

  python tools/seeded_slots_bench.py --workloads sobel harris --runs 2 --steps 20 --out DIR/seeded_slots.json
"""
import argparse
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

B, KEYSETS, BUDGET_TENANTS = 32, 8, 48
KERNELS = ("k_rot_wsum_ip", "k_rot_many", "k_ks_inner")


def outputs_equal(outs_a, outs_b, names):
    return all(np.array_equal(x.get(n)[1], y.get(n)[1]) for x, y in zip(outs_a, outs_b) for n in names)


MODES = ("expanded", "seeded")


def server(b200, params, **kw):
    return {m: b200.B200Server(params, hoist_constants="inline", key_storage=m, **kw) for m in MODES}


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
        nops = None
        wout = {}
        for keys in ("program", "power_of_two"):
            # a program holds its plans, and a plan the server it was built on: one program per group of servers, dropped with them
            prog = program_io.build_program(d)[0]
            srv = server(b200, params, capacity=B, rotation_keys=keys)
            elts = srv["expanded"].bank_info()["galois_elements"]
            keysets = [keys_for(elts, primes, N, 100 + s) for s in range(KEYSETS)]
            comp = [compressed(k, 1100 + i) for i, k in enumerate(keysets)]
            for s in srv.values():
                for t in range(B):
                    s.add_compressed_keys(*comp[t % KEYSETS])
                s.set_options(**opts)
            if nops is None:
                pub = b200.context_from_raw_keys(N, primes, *keysets[0])
                nops = pub.cipher_op_count(prog)
                del pub
            reqs = list(zip(range(B), vals))
            outs = {h: s.execute_batch(prog, reqs) for h, s in srv.items()}
            equal = outputs_equal(outs["expanded"], outs["seeded"], d["outputs"])
            s0 = main_stream.cuda_stream
            for s in srv.values():
                for r in range(2 * B):
                    s.stage_inputs(prog, [(r % B, vals[r % B])], s0, r)
            torch.cuda.synchronize()

            def res(h, steps):
                s = srv[h]
                return resident(lambda i, g, st: s.run_resident(prog, st, 1, g + B * (i % 2), [g]), steps)

            def e2e(h, steps):
                s = srv[h]
                return measure(lambda i: s.execute_batch_async(prog, reqs, i & 1), s.execute_batch_result, steps)

            def lat(h, reps):
                s, ts = srv[h], []
                for r in range(reps):
                    t0 = time.perf_counter()
                    s.execute(prog, r % B, vals[r % B])
                    ts.append(time.perf_counter() - t0)
                return float(np.median(ts))
            for h in srv:
                e2e(h, 2 * args.warmup); res(h, args.warmup); lat(h, args.warmup)
            rate = {"resident": {h: [] for h in srv}, "e2e": {h: [] for h in srv}, "latency_ms": {h: [] for h in srv}}
            for r in range(args.runs):
                for h in (MODES if r % 2 == 0 else MODES[::-1]):
                    rate["resident"][h].append(round(B * nops / res(h, args.steps)))
                    rate["e2e"][h].append(round(B * nops * args.steps / e2e(h, args.steps)))
                    rate["latency_ms"][h].append(round(lat(h, args.steps) * 1e3, 3))
            # per-kernel device time of one 32-instance step, each mode in a profiled pass of its own
            from torch.profiler import ProfilerActivity, profile
            ktime = {}
            for h, s in srv.items():
                with profile(activities=[ProfilerActivity.CUDA]) as p:
                    s.execute_batch(prog, reqs)
                    torch.cuda.synchronize()
                ktime[h] = {k: 0.0 for k in KERNELS}
                for e in p.key_averages():
                    for k in KERNELS:
                        if k in e.key:
                            ktime[h][k] += e.device_time_total / 1e3   # ms per step
                ktime[h] = {k: round(v, 3) for k, v in ktime[h].items()}
            info = {h: {k: s.bank_info()[k] for k in ("tenant_bytes", "key_bytes_per_tenant", "indicator_bytes", "bank_bytes")}
                    for h, s in srv.items()}
            wout[keys] = {"outputs_equal": equal, "ops_per_s": rate, "kernel_ms_per_step": ktime, "bank": info,
                          "cipher_ops_per_instance": nops}
            print(wl, keys, json.dumps(wout[keys]), flush=True)
            del srv, prog, s
            gc.collect()
        # equal bank budget: 48 tenants, 32 distinct per step
        budget = int(args.budget_gb * 1e9)
        probe = {h: s.bank_info()["tenant_bytes"] for h, s in server(b200, params, capacity=1).items()}
        fit = {h: budget // probe[h] for h in probe}
        slots = {h: min(BUDGET_TENANTS, fit[h]) for h in probe}
        elts = b200.B200Server(params, capacity=1).bank_info()["galois_elements"]
        keysets = [keys_for(elts, primes, N, 200 + s) for s in range(KEYSETS)]
        comp = [compressed(k, 1200 + i) for i, k in enumerate(keysets)]
        prog = program_io.build_program(d)[0]
        srv = {}
        for h in MODES:   # max_tenants > slots: both servers page (the seeded one holds every tenant once filled)
            srv[h] = b200.B200Server(params, capacity=slots[h], max_tenants=BUDGET_TENANTS + 1, hoist_constants="inline", key_storage=h)
            for t in range(BUDGET_TENANTS):
                srv[h].add_compressed_keys(*comp[t % KEYSETS])
            srv[h].set_options(**opts)
        batch = lambda i: [((16 * i + g) % BUDGET_TENANTS, vals[g]) for g in range(B)]
        equal = True
        for i in range(2):
            o = {h: s.execute_batch(prog, batch(i)) for h, s in srv.items()}
            equal = equal and outputs_equal(o["expanded"], o["seeded"], d["outputs"])
        brate = {h: [] for h in srv}
        fills = {h: [] for h in srv}
        for h, s in srv.items():
            measure(lambda i: s.execute_batch_async(prog, batch(i), i & 1), s.execute_batch_result, 2 * args.warmup)
        for r in range(args.runs):
            for h in (MODES if r % 2 == 0 else MODES[::-1]):
                s = srv[h]
                f0 = s.bank_info()["fills"]
                dt = measure(lambda i: s.execute_batch_async(prog, batch(i), i & 1), s.execute_batch_result, args.steps)
                brate[h].append(round(B * nops * args.steps / dt))
                fills[h].append((s.bank_info()["fills"] - f0) / args.steps)
        # one fill: a 1-slot server with 2 tenants; a 1-instance call that alternates the tenants fills every time, one that repeats
        # a tenant never does.  The fill's time is the difference of their medians (host-timed, synchronous calls)
        one = {}
        for h, s1 in server(b200, params, capacity=1, max_tenants=2).items():
            for t in range(2):
                s1.add_compressed_keys(*comp[t])
            ts = {True: [], False: []}
            for r in range(2 * args.steps + 4):
                alt = r % 2 == 0
                tenant = (r // 2) % 2 if alt else s1.bank_info()["resident"][0]
                f0 = s1.bank_info()["fills"]
                t0 = time.perf_counter(); s1.execute_batch(prog, [(tenant, vals[0])]); dt = time.perf_counter() - t0
                if r >= 4:
                    ts[s1.bank_info()["fills"] > f0].append(dt)
            one[h] = {"fill_ms": round((float(np.median(ts[True])) - float(np.median(ts[False]))) * 1e3, 4) if ts[True] and ts[False] else None,
                      "calls": {str(k): len(v) for k, v in ts.items()}}
            del s1
        wout["equal_budget"] = {"one_fill": one,"budget_bytes": budget, "slots_in_budget": fit, "slots": slots, "tenants": BUDGET_TENANTS, "outputs_equal": equal,
                                "e2e_ops_per_s": brate, "fills_per_step": fills,
                                "bank_bytes": {h: s.bank_info()["bank_bytes"] for h, s in srv.items()}}
        print(wl, "equal_budget", json.dumps(wout["equal_budget"]), flush=True)
        del srv, prog, s
        gc.collect()
        result["workloads"][wl] = wout
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
