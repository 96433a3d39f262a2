"""Static SASS census of the N = 16384 fold transforms a Sobel execute launches (tools/ntt_sass_report.py): every variant is
in the built library, the butterflies stay below the instruction counts they had before the carry-chained fold products, and
the inverse transforms without a gather prologue keep spill code out of their butterfly passes.  Needs cuobjdump, not a GPU."""
import os
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
LIB = os.path.join(ROOT, "eva_b200", "lib", "libevab200.so")
CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")

# instructions per butterfly before fold_mul / fold61 / fold_canon took their addend through madc32 (sm_90a, CUDA 12.9)
BEFORE = {
    "k_ntt_fwd<14,PLAIN,STORE,8,1>": 25.07, "k_ntt_fwd<14,MODRED,STORE,8,1>": 25.86, "k_ntt_fwd<14,MODRED,STORE_LAZY,8,1>": 23.71,
    "k_ntt_fwd<14,MODRED,DIVROUND,8,1>": 29.79, "k_ntt_fwd<14,PLAIN,DIVROUND,8,1>": 29.43, "k_ntt_fwd<14,MODRED_SG,STORE_LAZY,8,1>": 25.5,
    "k_ntt_inv<14,PLAIN,STORE,8,1>": 27.57, "k_ntt_inv<14,PLAIN,ADDHALF,8,1>": 27.64, "k_ntt_inv<14,GATHER,STORE,8,1>": 28.21,
    "k_ntt_inv<14,PLAIN,STORE_ZFLAG,8,1>": 28.14,
}


@pytest.fixture(scope="module")
def rows():
    if not (os.path.exists(CUOBJDUMP) or shutil.which("cuobjdump")):
        pytest.skip("cuobjdump not available")
    import ntt_sass_report as r
    funcs = r.sass_functions(LIB)
    out = {}
    for name, ins in funcs.items():
        m = r.NAME.fullmatch(name)
        if m:
            out["k_ntt_%s<14,%s,%s,8,1>" % (m.group(1), r.PRO[int(m.group(2))], r.EPI[int(m.group(3))])] = r.census(ins)
    return out


def test_every_sobel_variant_is_built(rows):
    assert set(BEFORE) <= set(rows)


def test_fewer_instructions_per_butterfly(rows):
    for k, before in BEFORE.items():
        assert rows[k]["per_butterfly"] < before, (k, rows[k]["per_butterfly"], before)


def test_inverse_passes_spill_free(rows):
    for k in BEFORE:
        if k.startswith("k_ntt_inv") and "GATHER" not in k:
            assert rows[k]["spill_in_passes"] == 0, (k, rows[k])
