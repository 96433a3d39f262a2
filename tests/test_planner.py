"""The planner (eva_b200/csrc/host/planner.hpp) on its own, without a GPU: the plans of the fixture programs and the shipped
workloads under every scheduler and rewrite option, one-offset-per-value and packed.  Every read is ordered after the write
of what it reads (stream order plus event waits), every term step reads its program operands, and the arena layout keeps
values that are alive together apart.  The work sizes are stand-ins (the hook derives them from N and ell): these
invariants hold for any sizes; the GPU tests run the real ones."""
import glob
import json
import os
import re

import pytest

from eva_b200 import program_io as gl
from eva_b200._eva_b200 import _plan

from test_arena_packing import check_layout

PROGRAMS = sorted(os.path.basename(p)[:-5] for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "programs", "*.json"))
                  if "terms" in json.load(open(p)))   # (a fixture may record a compile error instead of a program)
PROGRAMS += ["sobel", "harris", "polynomial"]
OPTIONS = {
    "default": ({}, 1),
    "no_rotation_sums": (dict(rotation_sums=False), 1),
    "approx_hoist": (dict(approx_hoist=True), 1),
    "no_hoist_mod_up": (dict(hoist_mod_up=False), 1),
    "no_hoist": (dict(hoist_rotations=False), 1),
    "chunk1": (dict(rotation_chunk=1), 1),
    "chunk3": (dict(rotation_chunk=3), 1),
    "no_fuse_sums": (dict(fuse_sums=False), 1),
    "no_cache": (dict(cache_constants=False), 1),
    "no_dedup_terms": (dict(dedup_terms=False), 1),
    "streams1": (dict(num_streams=1), 1),
    "streams8": (dict(num_streams=8), 1),
    "batch2": ({}, 2),
}
_programs = {}


def program(name):
    if name not in _programs:
        d = gl.load_json(name)
        _programs[name] = (gl.build_program(d)[0], d["poly_modulus_degree"], len(d["prime_bits"]))
    return _programs[name]


def plan(name, opts, batch, limit=0):
    prog, N, k = program(name)
    return _plan(prog, N, k, dict(opts, arena_limit=limit), batch)


def happens_before(steps):
    """hb[i]: bit set of the steps ordered before step i, or step i itself (stream order plus event waits)"""
    recorder, hb, last = {}, [], {}
    for i, (_, _, stream, waits, record) in enumerate(steps):
        h = 1 << i
        if stream in last:
            h |= hb[last[stream]]
        for e in waits:
            assert e in recorder, "step %d waits on event %d, which no earlier step records" % (i, e)
            h |= hb[recorder[e]]
        hb.append(h)
        last[stream] = i
        if record >= 0:
            assert record not in recorder, "event %d recorded twice" % record
            recorder[record] = i
    return hb


def reads_of(p):
    reads = [set() for _ in p["steps"]]
    for r, (_, _, _, readers, _) in enumerate(p["regions"]):
        for i in readers:
            reads[i].add(r)
    return reads


def check_operands(p, prog, reads):
    """the regions a term step reads include those of its program operands.  An operand that is not materialised (absorbed
    into a fused sum, a rotation sum or a chunk's pseudo step) is followed to its own operands; what a rotation sum call
    reads counts for the fused sums it feeds"""
    terms = {t.index: t for t in prog.terms()}
    regions, values = p["regions"], p["values"]
    for i, (kind, index, _, _, _) in enumerate(p["steps"]):
        if kind != "Term":
            continue
        seen = set(reads[i])
        for r in reads[i]:
            w = regions[r][2]
            if w >= 0 and p["steps"][w][0] != "Term":
                seen |= reads[w]
        todo = list(terms[index].operands)
        while todo:
            o = todo.pop()
            if o.index in values:
                assert values[o.index][2] in seen, "step %d (t%d) does not read operand t%d" % (i, index, o.index)
            else:
                todo.extend(o.operands)


def check_plan(p, prog):
    steps, regions, values = p["steps"], p["regions"], p["values"]
    hb = happens_before(steps)
    reads = reads_of(p)
    for r, (words, off, writer, readers, pinned) in enumerate(regions):
        if writer < 0:   # not written by the run: inputs, cached constants, flags, workspaces, or never materialised
            assert pinned or not readers, "region %d is read but never written" % r
            continue
        for i in readers:
            assert i != writer and (hb[i] >> writer) & 1, "step %d reads region %d before its writer, step %d" % (i, r, writer)
    check_operands(p, prog, reads)
    for index, (off, words, r) in values.items():
        rw, ro = regions[r][0], regions[r][1]
        assert ro <= off and off + words <= ro + rw, "value t%d lies outside its region %d" % (index, r)
    if p["stats"]["packed"]:
        recorder = {st[4]: i for i, st in enumerate(steps) if st[4] >= 0}
        pack_steps = [(stream, sorted(recorder[e] for e in waits)) for _, _, stream, waits, _ in steps]
        check_layout(pack_steps, [(w, wr, rd, pn) for w, _, wr, rd, pn in regions], [r[1] for r in regions], [], p["stride"])
    else:
        spans = sorted((off, off + words) for words, off, _, _, _ in regions if words)
        for (a0, a1), (b0, b1) in zip(spans, spans[1:]):
            assert a1 <= b0, "regions [%d, %d) and [%d, %d) overlap" % (a0, a1, b0, b1)
        assert not spans or spans[-1][1] <= p["stride"]


@pytest.mark.parametrize("option", sorted(OPTIONS))
@pytest.mark.parametrize("name", PROGRAMS)
def test_plan_invariants(name, option):
    opts, batch = OPTIONS[option]
    prog = program(name)[0]
    p = plan(name, opts, batch)
    assert p["stats"]["packed"] == 0 and p["stats"]["arena_bytes"] == p["stats"]["arena_bytes_unpacked"]
    check_plan(p, prog)
    assert plan(name, opts, batch) == p
    limit = p["stats"]["arena_bytes_unpacked"] - 1
    try:
        q = plan(name, opts, batch, limit)
    except RuntimeError as e:   # nothing to reuse: the packed arena is as large as the unpacked one
        m = re.search(r"needs (\d+) bytes packed \((\d+) bytes unpacked\), more than the limit of (\d+)", str(e))
        assert m and int(m.group(1)) == int(m.group(2)) == limit + 1, e
        return
    assert q["stats"]["packed"] == 1 and q["stats"]["arena_bytes"] <= limit and q["stats"]["arena_bytes_unpacked"] == limit + 1
    check_plan(q, prog)
    assert plan(name, opts, batch, limit) == q
    below = q["stats"]["arena_bytes"] - 1
    with pytest.raises(RuntimeError, match=r"needs %d bytes packed \(%d bytes unpacked\), more than the limit of %d" % (below + 1, limit + 1, below)):
        plan(name, opts, batch, below)


def test_sobel_plan_is_one_rotation_sum_call():
    st = plan("sobel", {}, 1)["stats"]
    assert (st["rotation_sum_calls"], st["rotation_sums"], st["rotation_sum_rotations"], st["rotation_sum_taps"]) == (1, 2, 7, 1), st
    assert st["rotation_chunks"] == 0 and st["chunked_rotations"] == 0
