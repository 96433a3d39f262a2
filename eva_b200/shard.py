"""(Round-1 single-cut sharding, kept for its tests and helpers; the staged, device-resident successor is
eva_b200/dagshard.py.)  Sharding ONE compiled program across GPUs (SURVEY.md 8e; BASELINE configs "Harris 1->8 GPUs
DAG-sharded", "wide DAG across 8 GPUs").

Independent ciphertext ops of the DAG run on different GPUs and the only exchange is one final
gather (north_star: "NCCL only for the final gather"): the program is cut at its widest sum -- a
tree of cipher Add terms.  Modular addition is exact and associative, so the leaves of that tree can
be summed in any grouping with bit-identical results:

    part r   (rank r)   : the cones of the leaves assigned to r, ending in their partial sum
    tail     (rank 0)   : inputs partial_0 .. partial_{P-1} (gathered), their sum, then every term of
                          the original program that follows the cut (relinearize, rescale, outputs ...)

Terms shared by several cones (e.g. the rotations of the input) are recomputed by each part rather
than exchanged.  Everything below is host-side graph surgery on the IR through the same Program /
Term API the DSL uses; execution uses the ordinary executor on every rank.
"""
from . import Op, Program, Type

_ATTR_COPY = ("RescaleDivisorAttribute", "RangeAttribute", "EncodeAtScaleAttribute", "EncodeAtLevelAttribute", "TypeAttribute")


class Info:
    """static value information of a compiled term (the rules of the planner's value inference, planner.hpp / seal_executor.h)"""
    __slots__ = ("type", "size", "level", "scale")

    def __init__(self, type_, size, level, scale):
        self.type, self.size, self.level, self.scale = type_, size, level, scale


def infer(prog):
    """term index -> Info for every live term of a compiled program"""
    info = {}
    for t in prog.terms():
        a = t.attributes
        ops = [info[o.index] for o in t.operands]
        ciph = [i for i in ops if i.type == Type.Cipher]
        if t.op == Op.Input:
            ty = Type(a.get("TypeAttribute", Type.Cipher))
            info[t.index] = Info(ty, 2 if ty == Type.Cipher else 0, a.get("EncodeAtLevelAttribute", 0), a.get("EncodeAtScaleAttribute", 0))
        elif t.op == Op.Constant:
            info[t.index] = Info(Type.Raw, 0, 0, 0)
        elif t.op == Op.Encode:
            info[t.index] = Info(Type.Plain, 0, a["EncodeAtLevelAttribute"], a["EncodeAtScaleAttribute"])
        elif not ciph:
            ty = Type.Plain if any(i.type == Type.Plain for i in ops) else Type.Raw
            info[t.index] = Info(ty, 0, max([i.level for i in ops] + [0]), ops[0].scale if ops else 0)
        else:
            c0 = ciph[0]
            size, level, scale = max(i.size for i in ciph), max(i.level for i in ciph), c0.scale
            if t.op == Op.Mul:
                scale = sum(i.scale for i in ops if i.type != Type.Raw)
                if len(ciph) == 2:
                    size = ciph[0].size + ciph[1].size - 1
            elif t.op == Op.Relinearize:
                size = 2
            elif t.op == Op.Rescale:
                level, scale = level + 1, scale - a["RescaleDivisorAttribute"]
            elif t.op == Op.ModSwitch:
                level += 1
            info[t.index] = Info(Type.Cipher, size, level, scale)
    return info


def _add_trees(prog, info):
    """root term -> list of leaf terms, for every maximal tree of cipher+cipher Add terms"""
    terms = prog.terms()
    uses = {}
    for t in terms:
        for o in t.operands:
            uses[o.index] = uses.get(o.index, 0) + 1

    def cipher_add(t):
        return t.op == Op.Add and all(info[o.index].type == Type.Cipher for o in t.operands)

    absorbed, trees = set(), {}
    for root in reversed(terms):
        if not cipher_add(root) or root.index in absorbed:
            continue
        leaves = []
        stack = [(root, False)]          # iterative: an unbalanced chain of Adds may be thousands of terms deep
        while stack:
            t, inner = stack.pop()
            if cipher_add(t) and (not inner or uses.get(t.index, 0) == 1):
                if inner:
                    absorbed.add(t.index)
                for o in reversed(list(t.operands)):
                    stack.append((o, True))
            else:
                leaves.append(t)
        trees[root.index] = (root, leaves)
    return trees


def _clone(dst, memo, root, in_names):
    """copy term `root` (and its operands) of the source program into dst -- iterative, any depth"""
    stack = [root]
    while stack:
        t = stack[-1]
        if t.index in memo:
            stack.pop()
            continue
        pending = [o for o in t.operands if o.index not in memo]
        if pending:
            stack.extend(pending)
            continue
        stack.pop()
        args = [memo[o.index] for o in t.operands]
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
    """balanced tree of Add terms"""
    while len(xs) > 1:
        xs = [dst._make_term(Op.Add, [xs[i], xs[i + 1]]) if i + 1 < len(xs) else xs[i] for i in range(0, len(xs), 2)]
    return xs[0]


class ShardPlan:
    """parts[r]: Program computing output "partial"; tail: Program with inputs partial_<r>; partial_size:
    polynomials of a partial ciphertext; root_index: the term of the original program that was cut"""

    def __init__(self, parts, tail, partial_size, root_index, leaves_per_part, part_sizes=None):
        self.parts, self.tail, self.partial_size, self.root_index, self.leaves_per_part = parts, tail, partial_size, root_index, leaves_per_part
        # polynomials of each part's partial sum: a part holding only relinearized leaves sends 2, one with a raw product 3
        self.part_sizes = part_sizes or [partial_size] * len(parts)


def split_program(prog, nparts):
    """cut `prog` (compiled) at its widest cipher sum into `nparts` independent parts + a tail; returns
    None when the program has no sum with at least `nparts` leaves (nothing to shard)"""
    info = infer(prog)
    trees = _add_trees(prog, info)
    if nparts < 2 or not trees:
        return None
    root, leaves = max(trees.values(), key=lambda rl: len(rl[1]))
    if len(leaves) < nparts:
        return None
    in_names = {t.index: n for n, t in prog.inputs.items()}
    ri = info[root.index]
    # contiguous blocks of leaves (neighbouring leaves share rotations / sub-expressions most often)
    bounds = [round(i * len(leaves) / nparts) for i in range(nparts + 1)]
    parts = []
    for r in range(nparts):
        p = Program("%s.part%d" % (prog.name, r), prog.vec_size)
        memo = {}
        mine = [_clone(p, memo, leaf, in_names) for leaf in leaves[bounds[r]:bounds[r + 1]]]
        p._make_output("partial", _sum(p, mine))
        parts.append(p)
    tail = Program(prog.name + ".tail", prog.vec_size)
    partials = []
    for r in range(nparts):
        x = tail._make_input("partial_%d" % r, Type.Cipher)
        x._set_attributes({"EncodeAtScaleAttribute": ri.scale, "EncodeAtLevelAttribute": ri.level})
        partials.append(x)
    memo = {root.index: _sum(tail, partials)}
    out_names = {t.index: n for n, t in prog.outputs.items()}
    for t in prog.terms():
        if t.op == Op.Output:
            src = _clone(tail, memo, t.operands[0], in_names)
            o = tail._make_output(out_names[t.index], src)
            a = t.attributes
            if "RangeAttribute" in a:
                o._set_attributes({"RangeAttribute": a["RangeAttribute"]})
    part_sizes = [infer(p)[p.outputs["partial"].index].size for p in parts]
    return ShardPlan(parts, tail, ri.size, root.index, [bounds[r + 1] - bounds[r] for r in range(nparts)], part_sizes)


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


def run_part(pub, plan, rank, inputs):
    """rank `rank`'s share of the DAG: returns (partial ciphertext [size][ell][N], scale)"""
    _, partial, scale = pub.execute_full(plan.parts[rank], _subset(inputs, set(plan.parts[rank].inputs))).get("partial")
    return partial, scale


def run_tail(pub, plan, partials, scale, inputs):
    """rank 0: sum of the gathered partial ciphertexts and everything after the cut"""
    pub.set_input_sizes({"partial_%d" % r: int(p.shape[0]) for r, p in enumerate(partials)})   # each part's own size (2 or 3)
    tail_inputs = _subset(inputs, set(plan.tail.inputs))
    for r, p in enumerate(partials):
        tail_inputs.set_cipher("partial_%d" % r, p, scale)
    try:
        return pub.execute_full(plan.tail, tail_inputs)
    finally:
        pub.set_input_sizes({})


def execute_sharded(pub, prog, inputs, rank=0, world=1, plan=None, device=None):
    """every rank calls this with the same program and inputs (replicated, like the keys): rank r runs
    part r, the partial sums are gathered on rank 0 (the only exchange: NCCL, or gloo on CPU tensors),
    rank 0 runs the tail and returns the outputs (other ranks return None).  Bit-identical to
    pub.execute(prog, inputs) with compact_outputs off: the sharded modes ignore that option and return full ciphertexts."""
    from . import multi
    plan = plan or split_program(prog, world)
    if world == 1 or plan is None:
        return pub.execute_full(prog, inputs) if rank == 0 else None
    import os
    import time
    t0 = time.perf_counter()
    partial, scale = run_part(pub, plan, rank, inputs)
    t1 = time.perf_counter()
    gathered = multi.gather_outputs(partial, rank, world, device=device)
    t2 = time.perf_counter()
    out = run_tail(pub, plan, gathered, scale, inputs) if rank == 0 else None
    if os.environ.get("EVAB_TRACE"):
        print("[evab] sharded rank %d: part %.3f ms, gather %.3f ms, tail %.3f ms" % (rank, (t1 - t0) * 1e3, (t2 - t1) * 1e3, (time.perf_counter() - t2) * 1e3), flush=True)
    return out
