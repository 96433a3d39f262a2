"""The cost of a packed plan arena (DESIGN §2): bench.py's device-resident measurement of one workload, run with the
default layout and with every plan's arena limited to one byte below its unpacked size (or to --arena-limit BYTES),
alternating, so that both layouts see the same machine state.

    python tools/arena_bench.py [--workload sobel|harris] [--steps 20] [--warmup 3] [--repeat 2]

Prints one JSON line: the GPU's name and power limit, ops/s and ms per step of each run of each layout, and the
packed plan's arena_bytes, arena_bytes_unpacked and reuse_waits (the write-after-read waits the packing added)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402


def bench_args(a):
    """bench.py's defaults (single GPU, cached-constant encoding off as in every reported line)"""
    return argparse.Namespace(instances=a.instances, fuse=1, streams=8, no_graph=False, no_const_cache=True, no_dedup=False,
                              approx_hoist=False, rotation_chunk=16, warmup=a.warmup, dump_outputs=None, workload=a.workload)


def unpacked_bytes(workload):
    from eva_b200 import b200, program_io
    d = bench.load_workload(workload)
    N = d["poly_modulus_degree"]
    primes = b200.create_coeff_modulus(N, d["prime_bits"])
    relin, galois, _ = bench.synthetic_inputs(d, primes, seed=1)
    pub = b200.context_from_raw_keys(N, primes, relin, galois, 0)
    pub.set_options(cache_constants=False)
    prog, _, _, _ = program_io.build_program(d)
    return pub, prog, pub.plan_stats(prog)["arena_bytes_unpacked"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="sobel")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--instances", type=int, default=32)
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--arena-limit", type=int, default=0, metavar="BYTES", help="default: one byte below the unpacked arena of one plan")
    a = ap.parse_args()
    import torch
    from eva_b200 import b200
    torch.cuda.set_device(0)
    pub, prog, unpacked = unpacked_bytes(a.workload)
    limit = a.arena_limit or unpacked - 1
    pub.set_options(cache_constants=False, arena_limit=limit)
    stats = pub.plan_stats(prog)
    del pub, prog
    orig = b200.B200Public.set_options
    runs = {"unpacked": [], "packed": []}
    try:
        for _ in range(a.repeat):
            for layout in ("unpacked", "packed"):
                lim = limit if layout == "packed" else 0
                b200.B200Public.set_options = lambda self, _lim=lim, **kw: orig(self, **kw, arena_limit=_lim)
                r, _, _ = bench.measure_workload(bench_args(a), a.workload, a.steps, 0, 1, 0)
                runs[layout].append({"value": r["value"], "ms_per_step": r["ms_per_step"], "e2e_value": r["e2e"]["value"]})
    finally:
        b200.B200Public.set_options = orig
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"workload": a.workload, "gpu": gpu, "unit": "ops/s", "steps": a.steps, "instances": a.instances, "arena_limit": limit,
                      **{k: stats[k] for k in ("packed", "arena_bytes", "arena_bytes_unpacked", "reuse_waits")}, "runs": runs}))


if __name__ == "__main__":
    main()
