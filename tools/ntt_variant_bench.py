"""ntt_variant_bench.py -- where a Sobel step's device time goes, and what the N = 16384 transforms cost, on one GPU.

  batched   k_ntt_fwd / k_ntt_inv (PLAIN, STORE) at bench.py's roofline shape: one launch of 8192 residues of N = 16384 over
            4 primes of 60 bits (1 GiB footprint, far above L2), CUDA events over --iters launches after 3 warm-up launches
  step      one torch.profiler pass (a run of its own, graphs off so that every kernel is recorded) of a bench-shaped Sobel
            step: 32 instances, fuse 1, 8 streams.  Per kernel instantiation: launches, device time per step and per launch
            (the plan's launch shapes: mod-up with diagonal exits, mod-down with DIVROUND, rescale ...); per kernel family:
            share of the step's device time

The GPU name, power limit and max SM clock are read in the same call.

  python tools/ntt_variant_bench.py [--iters 20] [--out DIR/ntt_variant.json]
"""
import argparse
import collections
import ctypes as C
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from tenant_paging_bench import gpu_info  # noqa: E402

PRO = {"0": "PLAIN", "1": "MODRED", "2": "GATHER", "3": "MODRED_SG"}
EPI = {"0": "STORE", "1": "ADDHALF", "2": "DIVROUND", "3": "STORE_LAZY", "4": "STORE_ZFLAG"}


def batched(iters):
    import torch
    from eva_b200 import b200, cabi
    lib = cabi.load()
    N, L = 16384, 4
    pa = np.array(b200.create_coeff_modulus(N, [60] * L)[:L], dtype=np.uint64)
    h = C.c_void_p()
    assert lib.evab_ctx_create(N, pa.ctypes.data_as(cabi.u64p), L, torch.cuda.current_device(), C.byref(h)) == 0
    cnt = (1 << 30) // (N * 8)
    data = torch.randint(0, 1 << 59, (cnt, N), dtype=torch.int64, device="cuda")
    pidx = (C.c_int * L)(*range(L))
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = {}
    for name, fn in (("fwd", lib.evab_ntt_fwd), ("inv", lib.evab_ntt_inv)):
        for _ in range(3):
            assert fn(h, C.c_void_p(data.data_ptr()), cnt, pidx, L, st) == 0
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn(h, C.c_void_p(data.data_ptr()), cnt, pidx, L, st)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        out[name] = {"residues": cnt, "launch_ms": round(ms, 4), "ns_per_residue": round(ms * 1e6 / cnt, 1),
                     "GB_s_algorithmic": round(2.0 * cnt * N * 8 / (ms * 1e-3) / 1e9, 1)}
    del data
    lib.evab_ctx_destroy(h)
    return out


def short_name(key):
    m = re.search(r"k_ntt_(fwd|inv)<(\d+), (\d+), (\d+), (\d+), (\d+)>", key)
    if m:
        d, n, p, e, cl, ar = m.groups()
        return "k_ntt_%s<%s,%s,%s,%s,%s>" % (d, n, PRO.get(p, p), EPI.get(e, e), cl, ar)
    return re.sub(r"\(.*", "", key).replace("void ", "")


def family(name):
    for f in ("k_ntt_fwd", "k_ntt_inv", "k_rot_wsum_ip", "k_rot_many", "k_ks_inner", "k_lazy_rotsum", "k_dyadic", "k_mul_ct",
              "k_mul_plain", "k_sum_terms", "k_enc_", "k_scale_c0", "k_rot_wsum"):
        if name.startswith(f):
            return f.rstrip("_")
    return "other"


def profiled_step(instances):
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from eva_b200 import b200, program_io
    d = bench.load_workload("sobel")
    N = d["poly_modulus_degree"]
    primes = b200.create_coeff_modulus(N, d["prime_bits"])
    relin, galois, _ = bench.synthetic_inputs(d, primes, seed=1234)
    pub = b200.context_from_raw_keys(N, primes, relin, galois, 0)
    pub.set_options(num_streams=8, use_graph=False, cache_constants=False, fuse=1)
    prog = program_io.build_program(d)[0]
    vals = []
    for i in range(instances):
        _, _, cts = bench.synthetic_inputs({**d, "terms": []}, primes, seed=bench.multi_seed(0, i))
        v = b200.B200Valuation()
        for name, (ct, scale) in cts.items():
            v.set_cipher(name, ct, scale)
        vals.append(v)
    for _ in range(3):
        pub.execute_batch(prog, vals)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        pub.execute_batch(prog, vals)
        torch.cuda.synchronize()
    per = collections.defaultdict(lambda: [0, 0.0])
    for e in p.key_averages():
        if e.device_time_total <= 0:
            continue
        k = short_name(e.key)
        per[k][0] += e.count
        per[k][1] += e.device_time_total   # us
    total = sum(t for _, t in per.values())
    kernels = {k: {"launches": n, "us_per_step": round(t, 1), "us_per_launch": round(t / n, 2), "share": round(t / total, 4)}
               for k, (n, t) in sorted(per.items(), key=lambda kv: -kv[1][1])}
    fam = collections.Counter()
    for k, (_, t) in per.items():
        fam[family(k)] += t
    return {"instances": instances, "device_us_per_step": round(total, 1), "kernels": kernels,
            "families": {f: round(t / total, 4) for f, t in fam.most_common()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--instances", type=int, default=32)
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    res = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0), "batched": batched(args.iters)}
    print(json.dumps(res), flush=True)
    if not args.no_profile:
        res["step"] = profiled_step(args.instances)
        print(json.dumps(res["step"]["families"]), flush=True)
        for k, v in list(res["step"]["kernels"].items())[:30]:
            print("%-44s %s" % (k, json.dumps(v)), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
