"""Program keys against power-of-two keys on one GPU.  Two arms, alternating within each run (--runs):

  program        a Galois key for every rotation step of the program (generate_keys(rotation_keys="program"), today's default)
  power_of_two   a key for every NAF term of the program's steps; the other rotations are composed from them (SEAL's rotate_vector)

Measured per workload, with keys and ciphertexts of uniform residues (valid evaluator inputs, seeded):

  resident_ops_per_s   device-resident: every instance staged once on a plan replica of its own (fuse 1, its own stream), CUDA events
                       around each step of all instances, L2 flushed between steps (as tools/tenant_paging_bench.py); median step
  latency_ms           one instance alone: events around one run_resident of a batch-1 plan, median of --steps runs
  bank                 B200Server(rotation_keys=...) layout: bytes of one tenant's device region, tenants that fit in --budget-gb of
                       device slots, host bytes of a paged tenant, full and compressed
  one_fill             one paged fill of a tenant (tools/tenant_paging_bench.fill_costs: key upload + hoist constants; compressed:
                       c0 upload + expansion + constants), CUDA events

The GPU name and power limit are read in the same run.

  python tools/rotation_keys_bench.py --workloads sobel harris wide4096 --runs 2 --steps 20 --out DIR/rotation_keys.json
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from tenant_paging_bench import fill_costs, gpu_info, keys_for, uniform  # noqa: E402

ARMS = ("program", "power_of_two")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["sobel", "harris", "wide4096"])
    ap.add_argument("--instances", type=int, default=32, help="instances per step (Sobel, Harris)")
    ap.add_argument("--wide-instances", type=int, default=4, help="instances per step of wide4096 (its arena is large)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--budget-gb", type=float, default=64.0, help="device memory given to key-bank slots, for tenants per budget")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from eva_b200 import b200, program_io
    from eva_b200._eva_b200 import _rotation_key_steps
    main_stream = torch.cuda.current_stream()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > the 50 MB L2
    result = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0), "steps": args.steps, "runs": args.runs, "workloads": {}}
    print(result["gpu"], flush=True)
    for wl in args.workloads:
        d = program_io.load_json(wl)
        N = d["poly_modulus_degree"]
        prog, params, _, _ = program_io.build_program(d)
        primes = b200.create_coeff_modulus(N, d["prime_bits"])
        k = len(primes)
        B = args.wide_instances if wl.startswith("wide") else args.instances
        rng = np.random.default_rng(7)
        vals = []
        for _ in range(B):
            v = b200.B200Valuation()
            for name, info in d["signature"].items():
                v.set_cipher(name, uniform(rng, primes, (2,), k - 1 - info["level"], N), 2.0 ** info["scale"])
            vals.append(v)
        streams = [torch.cuda.Stream() for _ in range(B)]
        ctx, elts, keys = {}, {}, {}
        for arm in ARMS:
            elts[arm] = b200.B200Server(params, capacity=1, rotation_keys=arm).bank_info()["galois_elements"]
            assert len(elts[arm]) == len(set(_rotation_key_steps(params, arm)))
            keys[arm] = keys_for(elts[arm], primes, N, 11)
            pub = b200.context_from_raw_keys(N, primes, *keys[arm])
            pub.set_options(fuse=1)
            ctx[arm] = pub
        nops = ctx["program"].cipher_op_count(prog)
        assert ctx["power_of_two"].cipher_op_count(prog) == nops
        s0 = main_stream.cuda_stream
        for arm in ARMS:
            for g in range(B):
                ctx[arm].stage_inputs(prog, [vals[g]], s0, g)
            ctx[arm].stage_inputs(prog, [vals[0]], s0, B)   # the latency replica
        torch.cuda.synchronize()

        def resident(arm, steps):
            pub = ctx[arm]
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
            for i in range(steps):
                flush.zero_()
                ev[i][0].record(main_stream)
                fork = torch.cuda.Event()
                fork.record(main_stream)
                for g in range(B):
                    streams[g].wait_event(fork)
                    pub.run_resident(prog, streams[g].cuda_stream, 1, g)
                    e = torch.cuda.Event()
                    e.record(streams[g])
                    main_stream.wait_event(e)
                ev[i][1].record(main_stream)
            torch.cuda.synchronize()
            return float(np.median([a.elapsed_time(b) for a, b in ev])) * 1e-3

        def latency(arm, steps):
            pub = ctx[arm]
            ts = []
            for _ in range(steps):
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(main_stream)
                pub.run_resident(prog, s0, 1, B)
                b.record(main_stream)
                b.synchronize()
                ts.append(a.elapsed_time(b))
            return float(np.median(ts))
        for arm in ARMS:
            resident(arm, max(3, args.warmup))
            latency(arm, max(3, args.warmup))
        rates = {a: [] for a in ARMS}
        lat = {a: [] for a in ARMS}
        for r in range(args.runs):
            for arm in (ARMS if r % 2 == 0 else ARMS[::-1]):
                rates[arm].append(B * nops / resident(arm, args.steps))
                lat[arm].append(latency(arm, args.steps))
        out = {"cipher_ops_per_instance": nops, "instances": B,
               "resident_ops_per_s": {a: [round(x) for x in v] for a, v in rates.items()},
               "resident_ops_per_s_median": {a: round(float(np.median(v))) for a, v in rates.items()},
               "latency_ms": {a: [round(x, 3) for x in v] for a, v in lat.items()},
               "latency_ms_median": {a: round(float(np.median(v)), 3) for a, v in lat.items()},
               "plan": {a: {s: ctx[a].plan_stats(prog, 1, 0)[s] for s in ("composed_rotations", "composed_hops", "hoist_groups", "rotation_chunks",
                                                                          "rotation_sum_calls", "steps", "arena_bytes")} for a in ARMS},
               "bank": {}, "one_fill": {}}
        for arm in ARMS:
            info = b200.B200Server(params, capacity=1, rotation_keys=arm).bank_info()
            nkeys = 1 + len(info["galois_elements"])
            out["bank"][arm] = {"galois_keys": len(info["galois_elements"]), "tenant_bytes": info["tenant_bytes"],
                                "tenants_per_budget": int(args.budget_gb * 2 ** 30 // info["tenant_bytes"]),
                                "host_bytes_full": nkeys * (k - 1) * 2 * k * N * 8, "host_bytes_compressed": nkeys * ((k - 1) * k * N * 8 + 32)}
        for r in range(args.runs):
            for arm in (ARMS if r % 2 == 0 else ARMS[::-1]):
                fc = fill_costs(N, primes, elts[arm], keys[arm])
                for key in ("fill_ms", "compressed_fill_together_ms"):
                    out["one_fill"].setdefault(arm, {}).setdefault(key, []).append(round(fc[key], 4))
        print(wl, json.dumps(out), flush=True)
        result["workloads"][wl] = out
        del ctx
        torch.cuda.synchronize()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
