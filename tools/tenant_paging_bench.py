"""Paged evaluation keys on one GPU: ops/s of a compiled workload (Sobel, Harris) with 32 instances per step (fuse 1), measured as
tools/tenant_bench.py measures -- device-resident (inputs staged once, one plan replica per instance on its own stream, CUDA events
around every step, L2 flushed between steps) and end to end with two steps in flight (execute_batch_async / execute_batch_result) --
under these arms, alternating within each run (--runs):

  no_paging        B200Server(capacity=32), 32 tenants resident             (the server without paging)
  paging_fit       B200Server(capacity=32, max_tenants=128), 32 tenants     (paging on, every tenant fits: no fill after warm-up)
  paging_miss_M    B200Server(capacity=32, max_tenants=128), 128 tenants; every step names 32 distinct tenants of which M are not
                   resident (M = 1, 8, 32): M fills per step, each waiting for the runs that read its slot

Every arm also runs with compressed tenants (suffix _c: add_compressed_keys, the c0 rows and a 32-byte seed per key; a fill uploads
the c0 rows and expands the c1 rows on the device), alternating with the full-key arms in the same run.

Also measured, with CUDA events on one stream: one fill split into the key upload (page-locked host -> device) and the hoist
constants (evab_rotate_hoist_const_levels), and one tenant's constants with the old loop of one evab_rotate_hoist_const call per
(element, level); and one compressed fill split into the c0 upload (one strided evab_upload_2d, and for comparison one
evab_upload per digit), the seed upload + expansion (evab_expand_key_uniform) and the constants.  Keys and ciphertexts are uniform residues (valid evaluator inputs), seeded.  The GPU name and power limit are
read in the same run.

  python tools/tenant_paging_bench.py --workloads sobel harris --runs 2 --steps 20 --out DIR/paging.json
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

SLOTS, TENANTS, KEYSETS = 32, 128, 8     # 128 tenants share 8 distinct key sets (their bytes do not change any cost)


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


def compressed(keys, seed):
    """add_compressed_keys arguments from a key set: its c0 rows and seeded 32-byte seeds"""
    rng = np.random.default_rng(seed)
    rk, gk = keys
    sd = lambda: rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
    return (np.ascontiguousarray(rk[:, 0]), sd(), {e: np.ascontiguousarray(v[:, 0]) for e, v in gk.items()}, {e: sd() for e in gk})


class Schedule:
    """steps of B distinct tenants, `misses` (M) of them not resident under the server's LRU policy (32 slots): positions M .. B-1
    keep tenants M .. B-1, positions 0 .. M-1 take the next M tenants of a round robin over all the others.  A batch touches its
    tenants in position order, so the tenants of positions 0 .. M-1 are the least recently used and exactly those are evicted by
    the next step's misses; the round robin (96 + M >= 2 M tenants) never returns to a tenant of the previous step"""

    def __init__(self, misses, B):
        self.misses, self.B, self.step = misses, B, 0
        self.pool = list(range(misses)) + list(range(B, TENANTS))

    def next(self):
        M, pool = self.misses, self.pool
        head = [pool[(self.step * M + g) % len(pool)] for g in range(M)]
        self.step += 1
        return head + list(range(M, self.B))


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


def fill_costs(N, primes, elts, keys, reps=10):
    """event-timed (ms): key upload of one tenant, its constants in one evab_rotate_hoist_const_levels call, and the same constants
    in one evab_rotate_hoist_const call per (element, level); the two agree word for word"""
    import torch
    from eva_b200 import cabi
    lib = cabi.load()
    k, n = len(primes), len(elts)
    pa = np.array(primes, dtype=np.uint64)
    h = C.c_void_p()
    assert lib.evab_ctx_create(C.c_uint64(N), pa.ctypes.data_as(C.POINTER(C.c_uint64)), k, 0, C.byref(h)) == 0
    for e in elts:
        assert lib.evab_galois_prepare(h, C.c_uint64(e)) == 0
    host = torch.from_numpy(np.concatenate([keys[0].ravel()] + [keys[1][e].ravel() for e in elts]).view(np.int64)).pin_memory()
    kw = keys[0].size
    dev = torch.empty_like(host, device="cuda")
    per = lib.evab_hoist_const_levels_bytes(h) // 8
    out, old = torch.empty(n * per, dtype=torch.int64, device="cuda"), torch.empty(n * per, dtype=torch.int64, device="cuda")
    tmp = torch.empty(lib.evab_rotate_hoist_const_levels_work_bytes(h, n) // 8, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream()
    sp = C.c_void_p(st.cuda_stream)
    ea = (C.c_uint64 * n)(*elts)
    gk = dev.data_ptr() + 8 * kw

    def levels():
        assert lib.evab_rotate_hoist_const_levels(h, n, ea, C.c_void_p(gk), C.c_void_p(out.data_ptr()), C.c_void_p(tmp.data_ptr()), sp) == 0

    def loop():
        off = 0
        for g, e in enumerate(elts):
            for ell in range(1, k):
                assert lib.evab_rotate_hoist_const(h, ell, C.c_uint64(e), C.c_void_p(gk + 8 * kw * g), C.c_void_p(old.data_ptr() + 8 * off),
                                                   C.c_void_p(tmp.data_ptr()), sp) == 0
                off += 2 * (ell + 1) * N

    def timed(fn):
        fn()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st); fn(); b.record(st)
            b.synchronize()
            ts.append(a.elapsed_time(b))
        return float(np.median(ts))
    r = {"upload_ms": timed(lambda: dev.copy_(host, non_blocking=True)), "constants_levels_ms": timed(levels),
         "constants_per_level_loop_ms": timed(loop), "per_level_calls": n * (k - 1), "key_upload_bytes": host.numel() * 8,
         "constants_bytes_written": n * per * 8}
    torch.cuda.synchronize()
    r["levels_equal_loop"] = bool(torch.equal(out, old))
    r["fill_ms"] = r["upload_ms"] + r["constants_levels_ms"]
    # compressed fill: the c0 rows of the n + 1 keys ((k-1) (n+1) rows of k N words, 2 k N words apart on the device)
    kN = k * N
    rows = (k - 1) * (n + 1)
    c0 = torch.from_numpy(np.concatenate([keys[0][:, 0].ravel()] + [keys[1][e][:, 0].ravel() for e in elts]).view(np.int64)).pin_memory()
    seeds = torch.from_numpy(np.random.default_rng(3).integers(0, 1 << 62, 4 * (n + 1), dtype=np.int64)).pin_memory()
    dseeds = torch.empty_like(seeds, device="cuda")
    hp, dp = c0.data_ptr(), dev.data_ptr()

    def up2d():
        assert lib.evab_upload_2d(h, C.c_void_p(dp), 2 * kN * 8, C.c_void_p(hp), kN * 8, kN * 8, rows, sp) == 0

    def per_digit():
        for i in range(rows):
            assert lib.evab_upload(h, C.c_void_p(dp + 16 * kN * i), C.c_void_p(hp + 8 * kN * i), kN * 8, sp) == 0

    def expand():
        dseeds.copy_(seeds, non_blocking=True)
        assert lib.evab_expand_key_uniform(h, n + 1, C.c_void_p(dseeds.data_ptr()), pa.ctypes.data_as(C.POINTER(C.c_uint64)), C.c_void_p(dp), sp) == 0

    r.update({"c0_upload_2d_ms": timed(up2d), "c0_upload_per_digit_ms": timed(per_digit), "c0_upload_bytes": c0.numel() * 8, "c0_rows": rows,
              "expand_ms": timed(expand), "expand_words_written": rows * kN})
    r["compressed_fill_ms"] = r["c0_upload_2d_ms"] + r["expand_ms"] + r["constants_levels_ms"]

    def fill_c():
        up2d(); expand(); levels()
    r["compressed_fill_together_ms"] = timed(fill_c)
    lib.evab_ctx_destroy(h)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["sobel", "harris"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--misses", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from eva_b200 import b200, program_io
    B = SLOTS
    opts = dict(num_streams=8, fuse=1)
    main_stream = torch.cuda.current_stream()
    streams = [torch.cuda.Stream() for _ in range(B)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # > the 50 MB L2

    def resident(run, steps):
        """median step time (s) of `steps` device-resident steps: run(i, g, stream) enqueues instance g of step i"""
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
    result = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0), "instances": B, "slots": SLOTS, "tenants_paged": TENANTS,
              "steps": args.steps, "options": opts, "workloads": {}}
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
        plain = b200.B200Server(params, capacity=SLOTS)
        elts = plain.bank_info()["galois_elements"]
        keysets = [keys_for(elts, primes, N, 100 + s) for s in range(KEYSETS)]
        for t in range(B):
            plain.add_raw_keys(*keysets[t % KEYSETS])
        fit = b200.B200Server(params, capacity=SLOTS, max_tenants=TENANTS)
        for t in range(B):
            fit.add_raw_keys(*keysets[t % KEYSETS])
        paged = b200.B200Server(params, capacity=SLOTS, max_tenants=TENANTS)
        for t in range(TENANTS):
            paged.add_raw_keys(*keysets[t % KEYSETS])
        ckeys = [compressed(ks, 500 + i) for i, ks in enumerate(keysets)]
        plain_c = b200.B200Server(params, capacity=SLOTS)
        fit_c = b200.B200Server(params, capacity=SLOTS, max_tenants=TENANTS)
        for t in range(B):
            plain_c.add_compressed_keys(*ckeys[t % KEYSETS])
            fit_c.add_compressed_keys(*ckeys[t % KEYSETS])
        paged_c = b200.B200Server(params, capacity=SLOTS, max_tenants=TENANTS)
        for t in range(TENANTS):
            paged_c.add_compressed_keys(*ckeys[t % KEYSETS])
        for s in (plain, fit, paged, plain_c, fit_c, paged_c):
            s.set_options(**opts)
        pub = b200.context_from_raw_keys(N, primes, *keysets[0])
        nops = pub.cipher_op_count(prog)
        del pub
        # assignments: the warm-up and every run of an arm continue one schedule, so that each step misses exactly M
        sched = {(m, c): Schedule(m, B) for m in args.misses for c in ("", "_c")}
        fixed = list(range(B))
        arms = {}
        for c, (p0, p1, p2) in (("", (plain, fit, paged)), ("_c", (plain_c, fit_c, paged_c))):
            arms.update({"no_paging" + c: (p0, None, c), "paging_fit" + c: (p1, None, c)})
            arms.update({"paging_miss_%d%s" % (m, c): (p2, m, c) for m in args.misses})

        def assign(m, c):
            return fixed if m is None else sched[(m, c)].next()

        def e2e(name, steps):
            srv, m, c = arms[name]
            batches = [assign(m, c) for _ in range(steps)]
            f0 = srv.bank_info()["fills"]
            dt = measure(lambda i: srv.execute_batch_async(prog, list(zip(batches[i], vals)), i & 1), srv.execute_batch_result, steps)
            return dt, (srv.bank_info()["fills"] - f0) / steps

        # device-resident: instance g of step i on replica g + 32 (i % 2) (a replica's tenant table is rewritten only after its run
        # two steps back); every replica staged once
        s0 = main_stream.cuda_stream
        for name, (srv, m, c) in arms.items():
            for r in range(2 * B):
                srv.stage_inputs(prog, [(fixed[r % B], vals[r % B])], s0, r)
        torch.cuda.synchronize()

        def res(name, steps):
            srv, m, c = arms[name]
            batches = [assign(m, c) for _ in range(steps)]
            f0 = srv.bank_info()["fills"]
            dt = resident(lambda i, g, st: srv.run_resident(prog, st, 1, g + B * (i % 2), [batches[i][g]]), steps)
            return dt, (srv.bank_info()["fills"] - f0) / steps
        for name in arms:   # plans, replicas, graphs, both submit slots, the page-locked pool
            e2e(name, 2 * max(3, args.warmup))
            res(name, max(3, args.warmup))
        e2e_rates = {k: [] for k in arms}
        res_rates = {k: [] for k in arms}
        fills = {k: {"e2e": [], "resident": []} for k in arms}
        for r in range(args.runs):
            for name in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                dt, fps = res(name, args.steps)
                res_rates[name].append(B * nops / dt)
                fills[name]["resident"].append(fps)
                dt, fps = e2e(name, args.steps)
                e2e_rates[name].append(B * nops * args.steps / dt)
                fills[name]["e2e"].append(fps)
        info, info_c = paged.bank_info(), paged_c.bank_info()
        out = {
            "cipher_ops_per_instance": nops,
            "resident_ops_per_s": {k: [round(x) for x in v] for k, v in res_rates.items()},
            "resident_ops_per_s_median": {k: round(float(np.median(v))) for k, v in res_rates.items()},
            "e2e_ops_per_s": {k: [round(x) for x in v] for k, v in e2e_rates.items()},
            "e2e_ops_per_s_median": {k: round(float(np.median(v))) for k, v in e2e_rates.items()},
            "fills_per_step": fills,
            "bank": {k: info[k] for k in ("device_slots", "max_tenants", "tenant_bytes", "key_bytes_per_tenant", "hoist_const_bytes_per_tenant",
                                          "bank_bytes", "host_key_bytes", "fills", "evictions")},
            "bank_compressed": {k: info_c[k] for k in ("host_key_bytes", "compressed_tenants", "fills", "evictions")},
            "one_fill": fill_costs(N, primes, elts, keysets[0]),
        }
        print(wl, json.dumps(out), flush=True)
        result["workloads"][wl] = out
        del plain, fit, paged, plain_c, fit_c, paged_c
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
