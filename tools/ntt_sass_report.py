#!/usr/bin/env python3
"""ntt_sass_report.py -- static SASS census of the N = 16384 fold transforms (LOGN 14, 8 CTAs per residue, AR = 1)
that a Sobel execute launches, per butterfly.  No GPU needed: it reads `cuobjdump -sass` of the built library.

One transform of N = 16384 points is 14 stages x N/2 butterflies over N/16 threads, i.e. 14 x 8 = 112 butterflies per
thread, so "per butterfly" = SASS instructions of the kernel / 112 (prologue, exchanges and epilogue included).
The `spill_in_passes` column counts LDL / STL between the first and the last fold product (the funnel shift that takes
S >> 61 in fold_mul), which is where a spill would sit on the critical path.

Usage: python tools/ntt_sass_report.py [library.so] [--json]     (default: eva_b200/lib/libevab200.so)"""
import collections
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRO = {0: "PLAIN", 1: "MODRED", 2: "GATHER", 3: "MODRED_SG"}
EPI = {0: "STORE", 1: "ADDHALF", 2: "DIVROUND", 3: "STORE_LAZY", 4: "STORE_ZFLAG"}
# the variants of a Sobel execute (launch_fwd_c / launch_inv_c with fold arithmetic at N = 16384)
FWD = [(0, 0), (1, 0), (1, 3), (1, 2), (0, 2), (3, 3)]
INV = [(0, 0), (0, 1), (2, 0), (0, 4)]
BFLY_PER_THREAD = 14 * 8
NAME = re.compile(r"_Z9k_ntt_(fwd|inv)ILi14ELi(\d)ELi(\d)ELi8ELi1EEv9NttLaunchx")


def sass_functions(path):
    nvdis = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    out = subprocess.run([nvdis if os.path.exists(nvdis) else "cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,6})\*/\s+(.*?)\s*;", line)
        if m and cur:
            funcs[cur].append(m.group(2))
    return funcs


def opcode(txt):
    t = txt.split()
    return t[1] if t[0].startswith("@") else t[0]


def census(ins):
    ops = [opcode(t) for t in ins]
    h = collections.Counter(ops)
    # fold_mul extracts S >> 61 with a funnel shift (shf.l.wrap): the first and last of those bracket the butterfly passes
    fm = [i for i, o in enumerate(ops) if o.startswith("SHF.L.W")]
    lo, hi = (fm[0], fm[-1]) if fm else (0, -1)
    spill_passes = sum(1 for o in ops[lo:hi + 1] if o.startswith(("LDL", "STL")))
    pick = lambda pred: sum(c for o, c in h.items() if pred(o))
    return {
        "instructions": len(ops),
        "per_butterfly": round(len(ops) / BFLY_PER_THREAD, 2),
        "IMAD.WIDE": pick(lambda o: o.startswith("IMAD.WIDE")),
        "IADD3": pick(lambda o: o.startswith("IADD3")),
        "IMAD_other": pick(lambda o: o.startswith("IMAD") and not o.startswith("IMAD.WIDE")),
        "LOP3+SHF": pick(lambda o: o.startswith(("LOP3", "SHF"))),
        "LDG": pick(lambda o: o.startswith("LDG")),
        "LDL+STL": pick(lambda o: o.startswith(("LDL", "STL"))),
        "spill_in_passes": spill_passes,
    }


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    lib = args[0] if args else os.path.join(ROOT, "eva_b200", "lib", "libevab200.so")
    funcs = sass_functions(lib)
    rows = []
    for name, ins in funcs.items():
        m = NAME.fullmatch(name)
        if not m:
            continue
        d, p, e = m.group(1), int(m.group(2)), int(m.group(3))
        if (p, e) not in (FWD if d == "fwd" else INV):
            continue
        r = {"kernel": "k_ntt_%s<14,%s,%s,8,1>" % (d, PRO[p], EPI[e])}
        r.update(census(ins))
        rows.append(r)
    rows.sort(key=lambda r: r["kernel"])
    if "--json" in sys.argv:
        print(json.dumps(rows, indent=1))
        return
    cols = ["instructions", "per_butterfly", "IMAD.WIDE", "IADD3", "IMAD_other", "LOP3+SHF", "LDG", "LDL+STL", "spill_in_passes"]
    print("%-40s " % "kernel" + " ".join("%10s" % c[:10] for c in cols))
    for r in rows:
        print("%-40s " % r["kernel"] + " ".join("%10s" % r[c] for c in cols))


if __name__ == "__main__":
    main()
