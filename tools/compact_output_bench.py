"""Compact responses on one GPU: what set_options(compact_outputs=p) does to response size, request rate, device time and accuracy.

- Response bytes per request, full and compact, computed from the output shapes (the compiled programs' output level, scale and
  declared range; backend.hpp compactShape) for Sobel, Harris and the polynomial at p = 10 and 20.
- End to end: a B200Server with 32 tenants runs 32 Sobel requests per step (fuse 1, 8 streams), two steps in flight
  (execute_batch_async / execute_batch_result, as bench.py measures), with the option off and at p = 10, the two arms
  alternating within each run (--runs).
- Device time of one evab_compact_ciphers call per chunk shape (1 and 32 values; the Sobel, Harris, polynomial and a two-prime
  shape), CUDA events around --launches back-to-back calls on one stream.
- Accuracy: for p in {8, 16, 24}, the worst |decrypt(compact) - decrypt(full)| over every slot of 8 Sobel and 8 Harris requests,
  as a fraction of 2^-p.
- With --parent DIR (a built tree of the parent commit): bench.py --gpus 1 run alternately from this tree and from DIR, the option
  off in both.

The GPU's name, power limit and max SM clock are read in the same run.

  python tools/compact_output_bench.py --runs 2 --steps 20 --parent PARENT_TREE --out DIR/compact.json
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
u64p = C.POINTER(C.c_uint64)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def workload(name):
    from eva_b200 import program_io
    prog, params, sig, _ = program_io.build_program(program_io.load_json(os.path.join(ROOT, "workloads", name + ".json")))
    return prog, params, sig


def inputs_for(sig, rng):
    return {n: list(rng.uniform(0.0, 0.2, sig.vec_size)) for n in sig.inputs}


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


def response_bytes(m, name):
    """per output: full and compact bytes at p = 10 and 20, from the output's shape"""
    from eva_b200 import b200
    prog, params, sig = workload(name)
    pub, sec = b200.generate_keys(params, seed=3)
    out = pub.execute(prog, sec.encrypt(inputs_for(sig, np.random.default_rng(1)), sig))
    N, primes = params.poly_modulus_degree, list(pub.primes())
    r = {"N": N}
    for o in out.names():
        kind, ct, scale = out.get(o)
        rng_bits = prog.outputs[o].attributes["RangeAttribute"]
        e = {"ell": int(ct.shape[1]), "scale_log2": float(np.log2(scale)), "range": rng_bits, "full": int(ct.nbytes)}
        for p in (10, 20):
            compact, shift, bits, _ = m._compact_shape(primes, ct.shape[1], scale, rng_bits, p, N)
            e["p%d" % p] = {"bits": bits, "shift": shift, "compact": bool(compact),
                            "bytes": 2 * ((N * bits + 63) // 64) * 8 if compact else int(ct.nbytes)}
        r[o] = e
    return r


def server_rates(runs, steps, warmup):
    from eva_b200 import b200
    prog, params, sig = workload("sobel")
    pub, sec = b200.generate_keys(params, seed=40)
    srv = b200.B200Server(params, capacity=B)
    tenants = [srv.add_keys(pub) for _ in range(B)]   # 32 tenants (one key set registered 32 times: the same work per tenant)
    rng = np.random.default_rng(7)
    rq = [(t, sec.encrypt(inputs_for(sig, rng), sig)) for t in tenants]
    arms = {"off": dict(num_streams=8, fuse=1), "p10": dict(num_streams=8, fuse=1, compact_outputs=10)}

    def e2e(arm, n):
        srv.set_options(**arms[arm])
        return measure(lambda i: srv.execute_batch_async(prog, rq, i & 1), srv.execute_batch_result, n)
    for arm in arms:
        e2e(arm, 2 * max(3, warmup))
    rates = {k: [] for k in arms}
    for r in range(runs):
        for arm in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
            rates[arm].append(B * steps / e2e(arm, steps))
    srv.set_options(**arms["p10"])
    outs = srv.execute_batch(prog, rq)
    kinds = sorted({o.get(n)[0] for o in outs for n in o.names()})
    spread = {k: (max(v) - min(v)) / float(np.median(v)) for k, v in rates.items()}
    med = {k: float(np.median(v)) for k, v in rates.items()}
    diff = (med["p10"] - med["off"]) / med["off"]
    return {"workload": "sobel", "tenants": B, "requests_per_step": B, "steps": steps, "runs": runs, "options": arms,
            "requests_per_s": {k: [round(x, 1) for x in v] for k, v in rates.items()},
            "requests_per_s_median": {k: round(v, 1) for k, v in med.items()},
            "relative_spread": {k: round(v, 4) for k, v in spread.items()},
            "p10_vs_off": round(diff, 4), "difference_exceeds_spread": bool(abs(diff) > max(spread.values())),
            "p10_output_kinds": kinds}


def device_times(launches, reps=10):
    """ms per evab_compact_ciphers call (median over reps of the mean over `launches` calls), per chunk shape"""
    import torch
    from eva_b200 import b200, cabi
    lib = cabi.load()
    shapes = [("sobel", 16384, [60] * 5, 1, 60, 37), ("harris", 16384, [60] * 5, 1, 60, 47), ("polynomial", 8192, [60] * 3, 1, 54, 54),
              ("two_primes", 16384, [60] * 5, 2, 95, 46)]
    res = {}
    for name, N, bits_list, ell, shift, bits in shapes:
        primes = np.array(b200.create_coeff_modulus(N, bits_list), dtype=np.uint64)
        h = C.c_void_p()
        assert lib.evab_ctx_create(C.c_uint64(N), primes.ctypes.data_as(u64p), len(primes), 0, C.byref(h)) == 0
        st = torch.cuda.current_stream()
        sp = C.c_void_p(st.cuda_stream)
        W = (N * bits + 63) // 64
        for n in (1, B):
            rng = np.random.default_rng(n)
            src = torch.from_numpy(rng.integers(0, 1 << 59, n * 2 * ell * N, dtype=np.int64)).cuda()
            dst = torch.empty(n * 2 * W, dtype=torch.int64, device="cuda")
            work = torch.empty(lib.evab_compact_work_bytes(h, n, ell) // 8, dtype=torch.int64, device="cuda")
            hs = (C.c_void_p * n)(*[src.data_ptr() + 8 * b * 2 * ell * N for b in range(n)])
            hd = (C.c_void_p * n)(*[dst.data_ptr() + 8 * b * 2 * W for b in range(n)])

            def call():
                assert lib.evab_compact_ciphers(h, n, hs, hd, ell, shift, bits, C.c_void_p(work.data_ptr()), sp) == 0, lib.evab_last_error()
            call()
            ts = []
            for _ in range(reps):
                a, b_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(st)
                for _ in range(launches):
                    call()
                b_.record(st)
                b_.synchronize()
                ts.append(a.elapsed_time(b_) / launches)
            res["%s_n%d" % (name, n)] = {"N": N, "ell": ell, "shift": shift, "bits": bits, "values": n, "ms_per_call": round(float(np.median(ts)), 4),
                                         "ms_min": round(float(np.min(ts)), 4), "calls_averaged": launches, "full_bytes": n * 2 * ell * N * 8,
                                         "compact_bytes": n * 2 * W * 8}
        torch.cuda.synchronize()
        lib.evab_ctx_destroy(h)
    return res


def accuracy():
    from eva_b200 import b200
    res = {}
    for name in ("sobel", "harris"):
        prog, params, sig = workload(name)
        pub, sec = b200.generate_keys(params, seed=9)
        rng = np.random.default_rng(2)
        encs = [sec.encrypt(inputs_for(sig, rng), sig) for _ in range(8)]
        pub.set_options(compact_outputs=0)
        full = [sec.decrypt(o, sig) for o in pub.execute_batch(prog, encs)]
        for p in (8, 16, 24):
            pub.set_options(compact_outputs=p)
            comp = [sec.decrypt(o, sig) for o in pub.execute_batch(prog, encs)]
            worst = max(float(np.max(np.abs(np.array(a[n]) - np.array(c[n])))) for a, c in zip(full, comp) for n in a)
            res["%s_p%d" % (name, p)] = {"worst_abs_error": worst, "fraction_of_2^-p": round(worst * 2.0 ** p, 4), "requests": 8}
    return res


def bench_alternating(parent, runs, steps, warmup):
    out = {"this": [], "parent": []}
    for r in range(runs):
        for arm in (("this", "parent") if r % 2 == 0 else ("parent", "this")):
            cwd = ROOT if arm == "this" else parent
            q = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup)], cwd=cwd,
                               capture_output=True, text=True)
            line = [l for l in q.stdout.splitlines() if l.startswith("{")][-1]
            d = json.loads(line)
            out[arm].append({"ops_per_s": d["value"], "e2e_ops_per_s": d["e2e"]["value"]})
    med = {k: float(np.median([x["ops_per_s"] for x in v])) for k, v in out.items()}
    out["median_ops_per_s"] = med
    out["this_vs_parent"] = round((med["this"] - med["parent"]) / med["parent"], 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--parent", default=None)
    ap.add_argument("--bench-runs", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from eva_b200 import _eva_b200 as m
    result = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0)}
    print(result["gpu"], flush=True)
    result["response_bytes"] = {w: response_bytes(m, w) for w in ("sobel", "harris", "polynomial")}
    print(json.dumps(result["response_bytes"]), flush=True)
    result["device_time"] = device_times(args.launches)
    print(json.dumps(result["device_time"]), flush=True)
    result["accuracy"] = accuracy()
    print(json.dumps(result["accuracy"]), flush=True)
    result["server_e2e"] = server_rates(args.runs, args.steps, args.warmup)
    print(json.dumps(result["server_e2e"]), flush=True)
    if args.parent:
        result["bench_py"] = bench_alternating(args.parent, args.bench_runs, 20, 5)
        print(json.dumps(result["bench_py"]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
