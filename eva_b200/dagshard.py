"""DAG-sharded execution of ONE compiled program over the GPUs of a box (SURVEY.md 8e; BASELINE configs
"Harris corner detector 1 -> 8 GPUs DAG-sharded" and "synthetic wide DAG (>= 4096 parallel ciphertext
multiplications) across 8 GPUs").

The reference runs independent terms of one program on different CPU threads with shared operands
(/root/reference/eva/common/multicore_program_traversal.h:55-79).  On GPUs operands are not shared, so the
DAG is cut where an exchange is cheapest and exact: at sums.  A tree of cipher Add terms can be summed in any
grouping with bit-identical results (modular addition is exact, commutative and associative), therefore

    stage s, rank r : the cones of the leaves assigned to r, ending in ONE partial sum per cut root;
    exchange        : the partial sums of every rank, gathered (NCCL) straight from one arena into the other
                      -- all-gather for an inner cut (every rank goes on), gather on rank 0 for the last one;
    next stage      : adds the gathered partials (that IS the cut value) and continues.

Several cuts at the same depth share one stage (Harris: the two 3x3 gradient sums, then the three 3x3
pooling sums).  A cut is taken only when a cost model says it pays: leaves are assigned so that expensive
shared sub-terms (rotations, relinearizations, ciphertext products) are SPLIT between the ranks rather than
recomputed -- leaves with the same expensive ancestors go to the same rank, and a full a x b grid of
two-ancestor leaves (the wide DAG: rot(x, i) * rot(y, j)) is blocked in two dimensions -- and the estimated
time saved must exceed the price of the exchange.  Everything here is host-side graph surgery through the
same Program / Term API the DSL uses; the stage programs run on the ordinary executor of every rank, their
partial ciphertexts never leave device memory.
"""
import os
import time

from . import Op, Program, Type
from .shard import infer, _add_trees, _ATTR_COPY

# rough relative single-instance costs (tools/op_throughput.py): only the ratios matter
_COST = {Op.RotateLeftConst: 7.0, Op.RotateRightConst: 7.0, Op.Relinearize: 9.0, Op.Rescale: 4.0, Op.ModSwitch: 1.5,
         Op.Mul: 3.0, Op.Add: 1.5, Op.Sub: 1.5, Op.Negate: 1.5, Op.Encode: 0.5}
_EXPENSIVE = (Op.RotateLeftConst, Op.RotateRightConst, Op.Relinearize)
EXCHANGE_US = 45.0     # one NCCL (all-)gather of a ciphertext per rank on NVSwitch + the stage boundary


def _cost(t, info):
    if info[t.index].type != Type.Cipher:
        return 0.0
    if t.op == Op.Mul and sum(1 for o in t.operands if info[o.index].type == Type.Cipher) == 2:
        return 4.0
    return _COST.get(t.op, 0.0)


def canonical(prog):
    """term index -> first identical term (same op, same attributes, same canonical operands).  The reference
    compiler does not share repeated sub-expressions -- its wide DAG holds 8192 rotation terms, 127 of them
    distinct -- and a duplicate is the same value, so plans, cost estimates and stage programs work on the
    representatives (the executor aliases duplicates as well: ExecOptions::dedupTerms)."""
    rep, seen = {}, {}
    for t in prog.terms():
        a = t.attributes
        if t.op in (Op.Input, Op.Output):
            rep[t.index] = t
            continue
        key = (int(t.op), a.get("RotationAttribute"), a.get("RescaleDivisorAttribute"), a.get("EncodeAtScaleAttribute"), a.get("EncodeAtLevelAttribute"),
               tuple(a["ConstantValueAttribute"]) if "ConstantValueAttribute" in a else None, tuple(rep[o.index].index for o in t.operands))
        rep[t.index] = seen.setdefault(key, t)
    return rep


_REP = {}     # program identity -> canonical map of the program being planned (set by plan_stages)


def _ops(t):
    rep = _REP.get("rep")
    return [rep[o.index] for o in t.operands] if rep else list(t.operands)


def _cone(t, stop):
    """indices of t and of everything it depends on, not descending below `stop` terms (iterative)"""
    seen, stack = set(), [t]
    while stack:
        u = stack.pop()
        if u.index in seen or u.index in stop:
            continue
        seen.add(u.index)
        stack.extend(_ops(u))
    return seen


def _clone(dst, memo, root, in_names):
    """copy `root` and its operands into dst (iterative: DAGs deeper than the recursion limit are fine);
    memo maps source term index -> Term of dst and is where cut values / inputs are substituted"""
    stack = [root]
    while stack:
        t = stack[-1]
        if t.index in memo:
            stack.pop()
            continue
        pending = [o for o in _ops(t) if o.index not in memo]
        if pending:
            stack.extend(pending)
            continue
        stack.pop()
        args = [memo[o.index] for o in _ops(t)]
        a = t.attributes
        if t.op == Op.Input:
            n = dst._make_input(in_names[t.index], Type(a.get("TypeAttribute", Type.Cipher)))
        elif t.op == Op.Constant:
            v = list(a["ConstantValueAttribute"])
            n = dst._make_uniform_constant(v[0]) if len(v) == 1 else dst._make_dense_constant(v)
        elif t.op == Op.RotateLeftConst:
            n = dst._make_left_rotation(args[0], a["RotationAttribute"])
        elif t.op == Op.RotateRightConst:
            n = dst._make_right_rotation(args[0], a["RotationAttribute"])
        else:
            n = dst._make_term(t.op, args)
        keep = {k: (Type(a[k]) if k == "TypeAttribute" else a[k]) for k in _ATTR_COPY if k in a and not (t.op == Op.Input and k == "TypeAttribute")}
        if keep:
            n._set_attributes(keep)
        memo[t.index] = n
    return memo[root.index]


def _sum(dst, xs):
    while len(xs) > 1:
        xs = [dst._make_term(Op.Add, [xs[i], xs[i + 1]]) if i + 1 < len(xs) else xs[i] for i in range(0, len(xs), 2)]
    return xs[0]


def _assign(leaf_sigs, nranks):
    """leaf -> rank.  leaf_sigs[i] = tuple of the expensive private ancestors of leaf i (sorted term indices).
    Leaves with equal signatures stay together; a full a x b grid of two-ancestor signatures is blocked in two
    dimensions (a/pa + b/pb distinct ancestors per rank instead of a + b/P); otherwise groups go, largest first,
    to the rank that needs the fewest new ancestors (ties: the least loaded)."""
    n = len(leaf_sigs)
    pairs = [s for s in leaf_sigs if len(s) == 2]
    if len(pairs) == n and n >= nranks:
        # two families (e.g. the rotations of x and those of y): 2-colour the ancestors along the pairs
        colour, adj = {}, {}
        for a, b in pairs:
            adj.setdefault(a, set()).add(b); adj.setdefault(b, set()).add(a)
        ok = True
        for start in adj:
            if start in colour:
                continue
            colour[start] = 0
            todo = [start]
            while todo and ok:
                u = todo.pop()
                for w in adj[u]:
                    if w not in colour:
                        colour[w] = 1 - colour[u]; todo.append(w)
                    elif colour[w] == colour[u]:
                        ok = False
        if ok:
            oriented = [(a, b) if colour[a] == 0 else (b, a) for a, b in pairs]
            A = sorted({p[0] for p in oriented}); B = sorted({p[1] for p in oriented})
            if len(A) * len(B) == n and len(set(oriented)) == n:
                best = None
                for pa in range(1, nranks + 1):
                    if nranks % pa == 0 and pa <= len(A) and nranks // pa <= len(B):
                        pb = nranks // pa
                        c = -(-len(A) // pa) + -(-len(B) // pb)
                        if best is None or c < best[0]:
                            best = (c, pa, pb)
                if best:
                    _, pa, pb = best
                    ia = {a: i * pa // len(A) for i, a in enumerate(A)}
                    ib = {b: j * pb // len(B) for j, b in enumerate(B)}
                    return [ia[p[0]] * pb + ib[p[1]] for p in oriented]
    groups = {}
    for i, s in enumerate(leaf_sigs):
        groups.setdefault(s, []).append(i)
    have = [set() for _ in range(nranks)]
    load = [0] * nranks
    out = [0] * n
    # empty signatures (cheap leaves) last: they only balance the load
    for s, members in sorted(groups.items(), key=lambda kv: (-len(kv[0]) * len(kv[1]), kv[1][0])):
        if s:
            r = min(range(nranks), key=lambda q: (len(set(s) - have[q]) * 1000 + load[q], q))
            have[r].update(s)
            for i in members:
                out[i] = r
            load[r] += len(members) + 10 * len(s)
        else:
            for i in members:
                r = min(range(nranks), key=lambda q: (load[q], q))
                out[i] = r
                load[r] += 1
    return out


class Stage:
    """roots: cut terms of the source program (indices); progs[r]: the program of rank r, with one output
    "partial_<root>" per root; nranks: ranks that contribute (the others idle through this stage);
    leaves[r]: number of leaves rank r sums; est_*: cost-model estimates in microseconds"""

    def __init__(self):
        self.roots, self.progs, self.nranks, self.leaves = [], [], 0, []
        self.est_single = self.est_sharded = 0.0


class StagePlan:
    def __init__(self, prog, nparts):
        self.source, self.nparts, self.stages, self.tail = prog, nparts, [], None
        self.partial_names = {}    # program name -> {input name: (root, rank)}
        self.input_sizes = {}      # partial input name -> polynomials

    def describe(self):
        return [{"roots": len(s.roots), "ranks": s.nranks, "leaves_per_rank": s.leaves, "est_single_us": round(s.est_single, 1),
                 "est_sharded_us": round(s.est_sharded, 1)} for s in self.stages]


def plan_stages(prog, nparts, exchange_us=EXCHANGE_US, force=False):
    """cut `prog` (compiled) into stages for `nparts` ranks; None when no cut pays (or nparts < 2).
    force=True keeps every candidate cut regardless of the cost model (tests)."""
    if nparts < 2:
        return None
    info = infer(prog)
    terms = prog.terms()
    byidx = {t.index: t for t in terms}
    rep = canonical(prog)
    _REP["rep"] = rep
    try:
        return _plan_stages(prog, nparts, exchange_us, force, info, terms, byidx, rep)
    finally:
        _REP.pop("rep", None)


def _plan_stages(prog, nparts, exchange_us, force, info, terms, byidx, rep):
    trees = {r: (root, [rep[l.index] for l in leaves]) for r, (root, leaves) in _add_trees(prog, info).items() if rep[r].index == r}
    in_names = {t.index: n for n, t in prog.inputs.items()}
    out_names = {t.index: n for n, t in prog.outputs.items()}
    order = {t.index: i for i, t in enumerate(terms)}
    # candidate cuts in topological order, with their depth in cuts
    cands = sorted((r for r, (_, lv) in trees.items() if len(lv) >= 2), key=lambda r: order[r])
    accepted, depth = [], {}
    plan = StagePlan(prog, nparts)
    stop_inputs = {t.index for t in terms if t.op == Op.Input}
    # group candidates by cut depth (number of accepted cuts below them), stage by stage
    remaining = list(cands)
    stage_no = 0
    while remaining:
        avail = set(stop_inputs) | set(accepted)
        # candidates whose cone contains no other remaining candidate
        ready = []
        for r in remaining:
            cone = _cone(byidx[r], avail)
            if not any(o != r and o in cone for o in remaining):
                ready.append(r)
        if not ready:
            break
        st = _build_stage(prog, info, byidx, trees, ready, avail, nparts, in_names, stage_no, plan, exchange_us, force)
        remaining = [r for r in remaining if r not in ready]
        if st is not None:
            plan.stages.append(st)
            accepted.extend(st.roots)
            stage_no += 1
    if not plan.stages:
        return None
    # tail (rank 0): everything after the last cuts
    tail = Program(prog.name + ".tail", prog.vec_size)
    memo = _cut_inputs(tail, plan, prog, info, accepted, byidx, set(stop_inputs) | set(accepted), [t for t in terms if t.op == Op.Output])
    for t in terms:
        if t.op == Op.Output:
            src = _clone(tail, memo, rep[t.operands[0].index], in_names)
            o = tail._make_output(out_names[t.index], src)
            if "RangeAttribute" in t.attributes:
                o._set_attributes({"RangeAttribute": t.attributes["RangeAttribute"]})
    plan.tail = tail
    return plan


def _cut_inputs(dst, plan, prog, info, cuts, byidx, avail, sinks):
    """memo for cloning into dst: every cut value that the cones of `sinks` reach becomes the sum of its gathered
    partials, which enter dst as inputs cut<root>_p<rank>"""
    need = set()
    for s in sinks:
        stack, seen = [s], set()
        while stack:
            u = stack.pop()
            if u.index in seen:
                continue
            seen.add(u.index)
            if u.index in cuts:
                need.add(u.index)
                continue
            stack.extend(_ops(u))
    memo = {}
    names = plan.partial_names.setdefault(dst.name, {})
    for c in sorted(need):
        st = next(s for s in plan.stages if c in s.roots)
        ri = info[c]
        parts = []
        for r in range(st.nranks):
            nm = "cut%d_p%d" % (c, r)
            x = dst._make_input(nm, Type.Cipher)
            x._set_attributes({"EncodeAtScaleAttribute": ri.scale, "EncodeAtLevelAttribute": ri.level})
            names[nm] = (c, r)
            parts.append(x)
        memo[c] = _sum(dst, parts)
    return memo


def _build_stage(prog, info, byidx, trees, roots, avail, nparts, in_names, stage_no, plan, exchange_us, force):
    # leaves of all roots of this stage, their private cones and expensive-ancestor signatures
    leaves = []   # (root, leaf term)
    for r in roots:
        for lf in trees[r][1]:
            leaves.append((r, lf))
    cones = [_cone(lf, avail) for _, lf in leaves]
    shared_all = set.intersection(*cones) if cones else set()
    # signature of a leaf: its expensive ancestors that other leaves need as well (what an assignment can share or split)
    count = {}
    for cn in cones:
        for i in cn:
            count[i] = count.get(i, 0) + 1
    sigs = []
    for cn in cones:
        sigs.append(tuple(sorted(i for i in cn - shared_all if count[i] > 1 and (byidx[i].op in _EXPENSIVE or _cost(byidx[i], info) >= 4.0))))
    nranks = min(nparts, min(len(trees[r][1]) for r in roots))
    if nranks < 2:
        return None
    assign = _assign(sigs, nranks)
    # every rank must hold at least one leaf of every root (its partial sum must exist): repair greedily
    for r in roots:
        idx = [i for i, (rr, _) in enumerate(leaves) if rr == r]
        for q in range(nranks):
            if not any(assign[i] == q for i in idx):
                donor = max(range(nranks), key=lambda d: sum(1 for i in idx if assign[i] == d))
                mv = next(i for i in idx if assign[i] == donor)
                assign[mv] = q
    cost = lambda ids: sum(_cost(byidx[i], info) for i in ids)
    union_all = set().union(*cones)
    per_rank = [set().union(*[cones[i] for i in range(len(leaves)) if assign[i] == q]) for q in range(nranks)]
    est_single = cost(union_all)
    est_sharded = max(cost(s) for s in per_rank) + exchange_us
    if not force and est_single - est_sharded <= 0:
        return None
    st = Stage()
    st.roots, st.nranks, st.est_single, st.est_sharded = list(roots), nranks, est_single, est_sharded
    st.leaves = [sum(1 for a in assign if a == q) for q in range(nranks)]
    cuts = [c for s in plan.stages for c in s.roots]
    for q in range(nranks):
        p = Program("%s.s%d.r%d" % (prog.name, stage_no, q), prog.vec_size)
        mine = [lf for i, (_, lf) in enumerate(leaves) if assign[i] == q]
        memo = _cut_inputs(p, plan, prog, info, cuts, byidx, avail, mine)
        for r in roots:
            mine_r = [_clone(p, memo, lf, in_names) for i, (rr, lf) in enumerate(leaves) if rr == r and assign[i] == q]
            p._make_output("partial_%d" % r, _sum(p, mine_r))
        st.progs.append(p)
    return st


def finalize_sizes(plan):
    """polynomial count of every partial (a rank that sums only relinearized leaves sends 2 polynomials, one that
    holds a raw product sends 3): consumers declare their inputs with the producer's size"""
    sizes = {}
    for st in plan.stages:
        for q, p in enumerate(st.progs):
            _declare(plan, p)
            pi = infer_with_sizes(p, plan.input_sizes)
            for r in st.roots:
                sizes[(r, q)] = pi[p.outputs["partial_%d" % r].index].size
        for pname, names in plan.partial_names.items():
            for nm, (c, r) in names.items():
                if (c, r) in sizes:
                    plan.input_sizes[nm] = sizes[(c, r)]
    return sizes


def infer_with_sizes(p, input_sizes):
    info = infer(p)
    # infer() assumes size-2 inputs; partial inputs may carry 3 polynomials: propagate through Adds
    names = {t.index: n for n, t in p.inputs.items()}
    for t in p.terms():
        if t.op == Op.Input and names.get(t.index) in input_sizes:
            info[t.index].size = input_sizes[names[t.index]]
        elif info[t.index].type == Type.Cipher and t.op in (Op.Add, Op.Sub, Op.Negate, Op.ModSwitch, Op.Rescale, Op.Output):
            ciph = [info[o.index] for o in t.operands if info[o.index].type == Type.Cipher]
            if ciph:
                info[t.index].size = max(i.size for i in ciph)
    return info


def _declare(plan, p):
    pass


# ------------------------------------------------------------------------------------------------- execution
def run_plain(plan, x):
    """plaintext semantics of the staged plan (tests, CPU): every rank's stage programs through `evaluate`,
    partial sums handed on exactly as the device path does"""
    from . import evaluate
    have = {}
    for st in plan.stages:
        for q, p in enumerate(st.progs):
            ins = {}
            for nm in p.inputs:
                ins[nm] = have[plan.partial_names[p.name][nm]] if nm in plan.partial_names.get(p.name, {}) else x[nm]
            out = evaluate(p, ins)
            for r in st.roots:
                have[(r, q)] = out["partial_%d" % r]
    ins = {}
    for nm in plan.tail.inputs:
        ins[nm] = have[plan.partial_names[plan.tail.name][nm]] if nm in plan.partial_names.get(plan.tail.name, {}) else x[nm]
    return evaluate(plan.tail, ins)


class _DevMem:
    """zero-copy view of device memory for torch.as_tensor (CUDA array interface)"""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes // 8,), "typestr": "<i8", "data": (int(ptr), False), "version": 2}


def _tensor(ptr, nbytes):
    import torch
    return torch.as_tensor(_DevMem(ptr, nbytes), device="cuda")


class ShardedRunner:
    """One rank's side of the staged execution.  Built once per (context, plan): the stage plans of this rank
    (arena + captured CUDA graph each), tensors aliasing the partial-sum slots of those arenas, and the
    schedule of collectives.  run(inputs) is then: H2D of the inputs this rank reads, and per stage one graph
    launch + one NCCL (all-)gather per cut root, issued on the current CUDA stream; nothing is staged through
    the host and nothing is allocated."""

    def __init__(self, pub, plan, rank, world):
        import torch
        self.torch, self.pub, self.plan, self.rank, self.world = torch, pub, plan, rank, world
        finalize_sizes(plan)
        pub.set_input_sizes(dict(plan.input_sizes))
        try:
            self.progs = [(st.progs[rank] if rank < st.nranks else None) for st in plan.stages] + ([plan.tail] if rank == 0 else [])
            self.io = {p.name: pub.io_pointers(p) for p in self.progs if p is not None}
        finally:
            pub.set_input_sizes({})
        self.bufs = {}
        self.subsets = {}
        consumers = {}     # root -> [program] of this rank reading its partials
        for p in self.progs:
            if p is not None:
                for nm, (c, r) in plan.partial_names.get(p.name, {}).items():
                    if p not in consumers.setdefault(c, []):
                        consumers[c].append(p)
        # static schedule: per stage, per root: (send tensor, optional pre-copy, recv tensor, gather?, post-copies)
        self.schedule = []
        for si, st in enumerate(plan.stages):
            p = self.progs[si]
            last = si == len(plan.stages) - 1
            ops = []
            for root in st.roots:
                sizes = [plan.input_sizes["cut%d_p%d" % (root, r)] for r in range(st.nranks)]
                cons = consumers.get(root, [])
                o = self.io[p.name]["outputs"]["partial_%d" % root] if p is not None else None
                if o is not None:
                    poly_bytes = o["bytes"] // o["size"]
                elif cons:
                    s0 = self._slots(cons[0], root, st.nranks)[0]
                    poly_bytes = s0["bytes"] // s0["size"]
                else:
                    poly_bytes = self._poly_bytes(root)
                nbytes, words = max(sizes) * poly_bytes, max(sizes) * poly_bytes // 8
                pre = None
                if o is not None and o["bytes"] == nbytes:
                    send = _tensor(o["ptr"], nbytes)
                else:     # idle rank, or fewer polynomials than the widest partial: through a zero-padded buffer
                    send = self._buf(("send", root), nbytes)
                    send.zero_()
                    if o is not None:
                        pre = (send[: o["bytes"] // 8], _tensor(o["ptr"], o["bytes"]))
                recv, direct = None, False
                need_recv = cons and (not last or rank == 0)
                if need_recv and all(sz == max(sizes) for sz in sizes) and st.nranks == world:
                    slots = self._slots(cons[0], root, st.nranks)
                    if all(slots[r + 1]["ptr"] - slots[r]["ptr"] == nbytes for r in range(st.nranks - 1)):
                        recv, direct = _tensor(slots[0]["ptr"], nbytes * world), True    # NCCL writes into the consumer's arena
                if recv is None and (not last or rank == 0 or len(st.roots) > 1):
                    recv = self._buf(("recv", root), nbytes * world)
                post = []
                for ci, cp in enumerate(cons):
                    if direct and ci == 0:
                        continue
                    for r, sl in enumerate(self._slots(cp, root, st.nranks)):
                        post.append((_tensor(sl["ptr"], sl["bytes"]), recv[r * words: r * words + sl["bytes"] // 8]))
                ops.append({"send": send, "pre": pre, "recv": recv, "words": words, "post": post, "direct": direct})
            self.schedule.append((p, last, ops))

    def _poly_bytes(self, root):
        """bytes of one polynomial of cut `root` for a rank that neither produces nor reads it (it still takes
        part in the collective with a zero buffer): ell residues of N coefficients at the cut's level"""
        ell = len(self.pub.primes()) - 1 - infer(self.plan.source)[root].level
        for io in self.io.values():
            for e in list(io["inputs"].values()) + list(io["outputs"].values()):
                if e is not None:
                    return e["bytes"] // e["size"] // e["ell"] * ell
        raise RuntimeError("rank %d holds no plan of the sharded program" % self.rank)

    def _slots(self, p, root, nranks):
        names = {v: k for k, v in self.plan.partial_names[p.name].items()}
        io = self.io[p.name]
        return [io["inputs"][names[(root, r)]] for r in range(nranks)]

    def _inputs_for(self, inputs):
        key = id(inputs)
        if key not in self.subsets:
            self.subsets.clear()
            self.subsets[key] = [(p, _subset(inputs, set(p.inputs) - set(self.plan.partial_names.get(p.name, {})))) for p in self.progs if p is not None]
        return self.subsets[key]

    def run(self, inputs, stream=None):
        torch, pub, rank, world = self.torch, self.pub, self.rank, self.world
        import torch.distributed as dist
        st_ptr = torch.cuda.current_stream().cuda_stream if stream is None else stream
        trace = os.environ.get("EVAB_TRACE")
        marks = [("start", time.perf_counter())]

        def mark(name):
            if trace:
                torch.cuda.synchronize()
                marks.append((name, time.perf_counter()))
        for p, sub in self._inputs_for(inputs):     # H2D of the source inputs into every stage arena that reads them
            if sub.names():
                pub.stage_inputs(p, [sub], st_ptr)
        mark("h2d")
        for si, (p, last, ops) in enumerate(self.schedule):
            if p is not None:
                pub.run_resident(p, st_ptr)
            mark("stage%d" % si)
            for op in ops:
                if op["pre"] is not None:
                    op["pre"][0].copy_(op["pre"][1])
            if world > 1:
                if last and len(ops) == 1:        # the final gather: only rank 0 (the tail) needs the partials
                    op = ops[0]
                    w = op["words"]
                    dist.gather(op["send"], [op["recv"][r * w:(r + 1) * w] for r in range(world)] if rank == 0 else None, dst=0)
                elif len(ops) == 1:
                    dist.all_gather_into_tensor(ops[0]["recv"], ops[0]["send"])
                else:           # several cut roots in one stage: ONE grouped NCCL launch for all of them
                    with dist._coalescing_manager(device=torch.device("cuda", torch.cuda.current_device())):
                        for op in ops:
                            dist.all_gather_into_tensor(op["recv"], op["send"])
            else:
                for op in ops:
                    op["recv"][: op["words"]].copy_(op["send"])
            for op in ops:
                for dst, src in op["post"]:
                    dst.copy_(src)
            mark("exchange%d" % si)
        out = None
        if rank == 0:
            pub.run_resident(self.plan.tail, st_ptr)
            mark("tail")
            out = pub.download_outputs(self.plan.tail, st_ptr)
            mark("d2h")
        if trace:
            print("[evab] sharded rank %d: " % rank + ", ".join("%s %.3f ms" % (n, (t - marks[i][1]) * 1e3) for i, (n, t) in enumerate(marks[1:])), flush=True)
        return out

    def _buf(self, key, nbytes):
        b = self.bufs.get(key)
        if b is None or b.numel() * 8 < nbytes:
            b = self.torch.zeros(nbytes // 8, dtype=self.torch.int64, device="cuda")
            self.bufs[key] = b
        return b[: nbytes // 8]


def _subset(inputs, names):
    from . import b200
    out = b200.B200Valuation()
    for name in inputs.names():
        if name in names:
            kind, arr, scale = inputs.get(name)
            if kind == "cipher":
                out.set_cipher(name, arr, scale)
            elif kind == "seeded_cipher":      # carried compressed: the instance that stages it expands c1
                out.set_seeded_cipher(name, arr, inputs.get_seed(name), scale)
            elif kind == "compact_cipher":     # a response, never an input
                raise ValueError("input %s is a compact response (compact_outputs): it can only be decrypted" % name)
            elif kind == "stored":             # the entry lives in one server's store; a B200Public has none
                raise ValueError("input %s is a reference to a stored ciphertext (handle %d): the sharded modes run on B200Public "
                                 "contexts, which have no store; send the ciphertext inline" % (name, arr))
            elif kind == "plain":
                out.set_plain(name, arr, scale)
            else:
                out.set_raw(name, list(arr))
    return out


def execute_local(pub, plan, inputs):
    """every rank's share of the staged plan run one after the other on THIS GPU, partial sums copied between
    the arenas on the device -- the single-process check that a plan reproduces execute(prog) bit for bit
    (tests; the multi-GPU path is ShardedRunner under torchrun)"""
    import torch
    finalize_sizes(plan)
    pub.set_input_sizes(dict(plan.input_sizes))
    try:
        st = torch.cuda.current_stream().cuda_stream
        partial = {}

        def feed(p):
            sub = _subset(inputs, set(p.inputs) - set(plan.partial_names.get(p.name, {})))
            pub.stage_inputs(p, [sub], st)
            pio = pub.io_pointers(p)
            for nm, (c, r) in plan.partial_names.get(p.name, {}).items():
                s = pio["inputs"][nm]
                _tensor(s["ptr"], s["bytes"]).copy_(partial[(c, r)][: s["bytes"] // 8])
            return pio
        for stg in plan.stages:
            for q, p in enumerate(stg.progs):
                pio = feed(p)
                pub.run_resident(p, st)
                for root in stg.roots:
                    o = pio["outputs"]["partial_%d" % root]
                    assert o["size"] == plan.input_sizes["cut%d_p%d" % (root, q)]
                    partial[(root, q)] = _tensor(o["ptr"], o["bytes"]).clone()
        feed(plan.tail)
        pub.run_resident(plan.tail, st)
        return pub.download_outputs(plan.tail, st)
    finally:
        pub.set_input_sizes({})


class AutoShardedRunner:
    """Sharding pays for wide programs (the 4096-product DAG: 4.7x on 8 GPUs) and not for short ones at small GPU counts
    (Harris: 0.95x on 2, 1.24x on 8): the cost model decides which cuts are candidates, a measurement decides whether the
    plan is used.  calibrate() times execute() on rank 0 against the staged run on all ranks (a few trials each, max over
    ranks) and every rank adopts rank 0's verdict; run() then takes the faster path.  Results are bit-identical either way."""

    def __init__(self, pub, prog, rank, world, plan=None):
        self.pub, self.prog, self.rank, self.world = pub, prog, rank, world
        self.plan = plan if plan is not None else plan_stages(prog, world)
        self.runner = ShardedRunner(pub, self.plan, rank, world) if self.plan is not None and world > 1 else None
        self.use_sharded = False
        self.timings = None

    def calibrate(self, inputs, trials=5):
        import torch
        import torch.distributed as dist
        if self.runner is None:
            return False
        def best(fn):
            ts = []
            for _ in range(trials + 1):
                dist.barrier()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
            return min(ts[1:])
        t_sh = torch.tensor([best(lambda: self.runner.run(inputs))], dtype=torch.float64, device="cuda")
        dist.all_reduce(t_sh, op=dist.ReduceOp.MAX)
        t_single = best(lambda: self.pub.execute_full(self.prog, inputs) if self.rank == 0 else None)
        verdict = torch.tensor([1 if (self.rank == 0 and t_sh.item() < 0.97 * t_single) else 0], dtype=torch.int64, device="cuda")
        dist.broadcast(verdict, src=0)
        self.use_sharded = bool(verdict.item())
        self.timings = {"sharded_ms": t_sh.item() * 1e3, "single_ms": t_single * 1e3 if self.rank == 0 else None}
        return self.use_sharded

    def run(self, inputs):
        if self.use_sharded:
            return self.runner.run(inputs)
        return self.pub.execute_full(self.prog, inputs) if self.rank == 0 else None
