"""The gain of exact weighted rotation sums (DESIGN §4, set_options(rotation_sums=...)): bench.py's device-resident measurement
of Sobel and Harris with the rotation sums off and on, alternating, so that both settings see the same machine state.  The
outputs of the last execute_batch step of every run are compared word for word across the settings.

    python tools/rotsum_bench.py [--workloads sobel,harris] [--steps 20] [--warmup 3] [--repeat 2]
    python tools/rotsum_bench.py --profile [--workloads sobel] [--out DIR]

Prints one JSON line: the GPU's name and power limit, and per workload the ops/s, ms per step, single-instance latency and
launches per step of every run of each setting, the plan's rotation-sum statistics and whether the outputs were identical.
--profile instead runs one device-resident step per setting under torch.profiler (CUDA activities) and prints the device time
per kernel; the traces are written under --out."""
import argparse
import filecmp
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

SETTINGS = ("off", "on")


def bench_args(a, workload, dump):
    """bench.py's defaults (single GPU, constants encoded inside every run as in every reported line)"""
    return argparse.Namespace(instances=a.instances, fuse=1, streams=8, no_graph=False, no_const_cache=True, no_dedup=False,
                              approx_hoist=False, rotation_chunk=16, warmup=a.warmup, dump_outputs=dump, workload=workload)


def with_rotation_sums(on):
    from eva_b200 import b200
    orig = b200.B200Public.set_options
    b200.B200Public.set_options = lambda self, **kw: orig(self, **kw, rotation_sums=on)
    return orig


def plan_stats(workload, on):
    from eva_b200 import b200, program_io
    d = bench.load_workload(workload)
    N = d["poly_modulus_degree"]
    primes = b200.create_coeff_modulus(N, d["prime_bits"])
    relin, galois, _ = bench.synthetic_inputs(d, primes, seed=1)
    pub = b200.context_from_raw_keys(N, primes, relin, galois, 0)
    pub.set_options(cache_constants=False, rotation_sums=on)
    prog, _, _, _ = program_io.build_program(d)
    st = pub.plan_stats(prog)
    return {k: st[k] for k in ("steps", "rotation_sum_calls", "rotation_sums", "rotation_sum_rotations", "rotation_sum_taps",
                               "chunked_rotations", "elided_rotations")}


def same_dirs(x, y):
    names = sorted(os.listdir(x))
    return names == sorted(os.listdir(y)) and all(filecmp.cmp(os.path.join(x, n), os.path.join(y, n), shallow=False) for n in names)


def measure(a):
    from eva_b200 import b200
    out = {}
    tmp = tempfile.mkdtemp(prefix="rotsum_bench_")
    for wl in a.workloads.split(","):
        runs = {s: [] for s in SETTINGS}
        dumps = []
        for rep in range(a.repeat):
            for s in SETTINGS:
                dump = os.path.join(tmp, "%s_%s_%d" % (wl, s, rep))
                orig = with_rotation_sums(s == "on")
                try:
                    r, _, _ = bench.measure_workload(bench_args(a, wl, dump), wl, a.steps, 0, 1, 0)
                finally:
                    b200.B200Public.set_options = orig
                runs[s].append({"value": r["value"], "ms_per_step": r["ms_per_step"], "latency_ms": r["single_instance"]["latency_ms"],
                                "launches_per_step": r["gpu_launches"] // a.steps})
                dumps.append(dump)
        out[wl] = {"runs": runs, "outputs_identical": all(same_dirs(dumps[0], d) for d in dumps[1:]),
                   "plan": {s: plan_stats(wl, s == "on") for s in SETTINGS}}
    return out


def profile(a):
    """one device-resident step of B instances (B concurrent single-instance graphs, as bench.py) per setting"""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    from eva_b200 import b200, program_io
    os.makedirs(a.out, exist_ok=True)
    out = {}
    for wl in a.workloads.split(","):
        d = bench.load_workload(wl)
        N = d["poly_modulus_degree"]
        primes = b200.create_coeff_modulus(N, d["prime_bits"])
        relin, galois, _ = bench.synthetic_inputs(d, primes, seed=1234)
        pub = b200.context_from_raw_keys(N, primes, relin, galois, 0)
        prog, _, _, _ = program_io.build_program(d)
        main = torch.cuda.current_stream()
        streams = [torch.cuda.Stream() for _ in range(a.instances)]
        for s in SETTINGS:
            pub.set_options(cache_constants=False, rotation_sums=s == "on")
            for g in range(a.instances):
                _, _, cts = bench.synthetic_inputs({**d, "terms": []}, primes, seed=bench.multi_seed(0, g))
                val = b200.B200Valuation()
                for name, (ct, scale) in cts.items():
                    val.set_cipher(name, ct, scale)
                pub.drop_plan(prog, 1, g)
                pub.stage_inputs(prog, [val], main.cuda_stream, g)

            def step():
                fork = torch.cuda.Event()
                fork.record(main)
                for g in range(a.instances):
                    streams[g].wait_event(fork)
                    pub.run_resident(prog, streams[g].cuda_stream, 1, g)
                    ev = torch.cuda.Event()
                    ev.record(streams[g])
                    main.wait_event(ev)
            for _ in range(3):
                step()
            torch.cuda.synchronize()
            with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
                step()
                torch.cuda.synchronize()
            prof.export_chrome_trace(os.path.join(a.out, "rotsum_%s_%s.json" % (wl, s)))
            kern = {}
            for e in prof.events():
                if e.device_type.name == "CUDA":
                    k = kern.setdefault(e.name, [0, 0.0])
                    k[0] += 1
                    k[1] += e.device_time
            total = sum(v[1] for v in kern.values())
            out.setdefault(wl, {})[s] = {"device_us": total, "kernels": sorted(([n, c, round(t, 1)] for n, (c, t) in kern.items()), key=lambda x: -x[2])}
        for g in range(a.instances):
            pub.drop_plan(prog, 1, g)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="sobel,harris")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--instances", type=int, default=32)
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--profile", action="store_true", help="per-kernel device time of one step per setting (torch.profiler)")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "rotsum_profile"), help="--profile: directory of the chrome traces")
    a = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    res = profile(a) if a.profile else measure(a)
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu, "unit": "ops/s", "steps": a.steps, "instances": a.instances, "results": res}))


if __name__ == "__main__":
    main()
