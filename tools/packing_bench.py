"""Slot packing on one GPU: requests per second of k = 1 (one request per ciphertext, the client replicating it to N/2 slots)
against the largest k (pack_program: k requests per ciphertext), at bench.py's shape -- 32 ciphertext instances per step, one
CUDA graph per instance on its own stream, 8 streams inside a plan, constants encoded inside every run.  Modes alternate within
each run (--runs).  Sobel and Harris (vec_size 4096, N = 16384) pack k = 2, the polynomial (vec_size 1024, N = 8192) k = 4.

  resident   inputs staged once; CUDA events around every step, L2 flushed between steps (untimed); median step
  e2e        execute_batch_async / execute_batch_result with two steps in flight, host buffers in and out (host wall clock)
  host       pack_inputs + unpack_outputs of one step's requests (numpy, host wall clock): the client's extra work
  mse        every request decrypted (and unpacked) against evaluate() of the unpacked program, on the same seeded inputs for both k

The GPU name, power limit and max SM clock are read in the same call.

  python tools/packing_bench.py --runs 2 --steps 20 --out DIR/packing.json
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from tenant_paging_bench import gpu_info, measure  # noqa: E402

B = 32   # ciphertext instances per step (bench.py --instances)
PACK = {"sobel": 2, "harris": 2, "polynomial": 4}
RANGE = {"sobel": (0.0, 0.2), "harris": (0.0, 0.2), "polynomial": (-1.0, 1.0)}


def requests(name, sig, n):
    """n requests, request j from seed j: the same inputs for every k"""
    lo, hi = RANGE[name]
    return [{nm: np.random.default_rng(1000 + j).uniform(lo, hi, sig.vec_size) for nm in sorted(sig.inputs)} for j in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=sorted(PACK))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from eva_b200 import b200, evaluate, program_io
    from eva_b200.ckks import pack_inputs, pack_program, unpack_outputs
    opts = dict(num_streams=8, use_graph=True, cache_constants=False, fuse=1)
    main_stream = torch.cuda.current_stream()
    streams = [torch.cuda.Stream() for _ in range(B)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def resident(pub, prog, steps):
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

    result = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0), "ciphertext_instances_per_step": B, "steps": args.steps,
              "runs": args.runs, "options": opts, "workloads": {}}
    print(result["gpu"], flush=True)
    for wl in args.workloads:
        kmax = PACK[wl]
        d = program_io.load_json(os.path.join(ROOT, "workloads", wl + ".json"))
        prog, params, sig, _ = program_io.build_program(d)
        reqs = requests(wl, sig, B * kmax)
        modes = {}
        for k in (1, kmax):
            p, pp, ps = pack_program(prog, params, sig, k)
            pub, sec = b200.generate_keys(pp, seed=3)
            pub.set_options(**opts)
            t0 = time.perf_counter()
            packed_in = [pack_inputs(reqs[i * k:(i + 1) * k], sig, k) for i in range(B)]
            t_pack = time.perf_counter() - t0
            vals = [pub.encrypt(x, ps) for x in packed_in]
            # every request once, for the MSE (k = 1: kmax batches of B)
            worst, total, outs_all = 0.0, 0.0, []
            for c in range(kmax // k):
                ins = vals if c == 0 else [pub.encrypt(pack_inputs(reqs[(c * B + i) * k:(c * B + i + 1) * k], sig, k), ps) for i in range(B)]
                for o in pub.execute_batch(p, ins):
                    outs_all.append(o)
            t0 = time.perf_counter()
            unpacked = [r for o in outs_all[:B] for r in unpack_outputs(sec.decrypt(o, ps), k)]
            t_unpack = time.perf_counter() - t0   # decryption included: the client's whole read-out of one step
            unpacked += [r for o in outs_all[B:] for r in unpack_outputs(sec.decrypt(o, ps), k)]
            assert len(unpacked) == len(reqs)
            for x, got in zip(reqs, unpacked):
                want = evaluate(prog, {n: list(v) for n, v in x.items()})
                for n in want:
                    m = float(np.mean((np.asarray(want[n]) - got[n]) ** 2))
                    worst, total = max(worst, m), total + m
            for g in range(B):
                pub.stage_inputs(p, [vals[g]], main_stream.cuda_stream, g)
            torch.cuda.synchronize()
            modes[k] = dict(prog=p, pub=pub, vals=vals, mse_max=worst, mse_mean=total / len(reqs), pack_ms=t_pack * 1e3,
                            decrypt_unpack_ms=t_unpack * 1e3, nops=pub.cipher_op_count(p))
        for k, m in modes.items():   # warm both paths
            resident(m["pub"], m["prog"], args.warmup)
            measure(lambda i: m["pub"].execute_batch_async(m["prog"], m["vals"], i & 1), m["pub"].execute_batch_result, 2 * args.warmup)
        rate = {"resident": {k: [] for k in modes}, "e2e": {k: [] for k in modes}}
        for r in range(args.runs):
            for k in (sorted(modes) if r % 2 == 0 else sorted(modes, reverse=True)):
                m = modes[k]
                dt = resident(m["pub"], m["prog"], args.steps)
                rate["resident"][k].append(round(B * k / dt, 1))
                dt = measure(lambda i: m["pub"].execute_batch_async(m["prog"], m["vals"], i & 1), m["pub"].execute_batch_result, args.steps)
                rate["e2e"][k].append(round(B * k * args.steps / dt, 1))
        med = {f: {k: float(np.median(v)) for k, v in rate[f].items()} for f in rate}
        wout = {"k_max": kmax, "vec_size": d["vec_size"], "N": d["poly_modulus_degree"],
                "requests_per_s": {f: {str(k): v for k, v in rate[f].items()} for f in rate},
                "gain": {f: round(med[f][kmax] / med[f][1], 3) for f in med},
                "cipher_ops_per_instance": {str(k): m["nops"] for k, m in modes.items()},
                "mse_vs_evaluate": {str(k): {"max": m["mse_max"], "mean": m["mse_mean"]} for k, m in modes.items()},
                "host_ms_per_step": {str(k): {"pack_inputs": round(m["pack_ms"], 3), "decrypt_and_unpack": round(m["decrypt_unpack_ms"], 3)}
                                     for k, m in modes.items()}}
        print(wl, json.dumps(wout), flush=True)
        result["workloads"][wl] = wout
        for k, m in modes.items():
            for g in range(B):
                m["pub"].drop_plan(m["prog"], 1, g)
        del modes
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
