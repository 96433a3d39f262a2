"""The arena packer (eva_b200/csrc/host/arena_packer.hpp) on its own, without a GPU: hand-written plans and seeded
random DAGs, each layout checked by an independent happens-before checker.  Two buffers may share words only if
every access of one (its writer and its readers) happens-before the writer of the other, where happens-before is
stream order plus the plan's waits plus the waits the packer added; pinned buffers overlap nothing."""
import random

import pytest

from eva_b200._eva_b200 import _pack_arena


def pack(steps, buffers):
    """steps: [(stream, [waited steps])]; buffers: [(words, writer, [readers], pinned)]"""
    offsets, waits, peak = _pack_arena(steps, buffers)
    check_layout(steps, buffers, offsets, waits, peak)
    return offsets, waits, peak


def happens_before(steps, extra_waits):
    """hb[i]: bit set of the steps that happen-before step i or are step i (transitive closure)"""
    waits = [list(w) for _, w in steps]
    for i, j in extra_waits:
        assert j < i, "an added wait must point to an earlier step"
        waits[i].append(j)
    hb, last = [], {}
    for i, (stream, _) in enumerate(steps):
        h = 1 << i
        if stream in last:
            h |= hb[last[stream]]
        for j in waits[i]:
            h |= hb[j]
        hb.append(h)
        last[stream] = i
    return hb


def check_layout(steps, buffers, offsets, waits, peak):
    hb = happens_before(steps, waits)
    assert len(offsets) == len(buffers)
    assert peak <= sum(b[0] for b in buffers)
    for k, (words, _, _, _) in enumerate(buffers):
        assert offsets[k] + words <= peak

    def ordered(a, b):   # every access of buffer a happens strictly before the writer of buffer b
        wb = buffers[b][1]
        return all(x != wb and (hb[wb] >> x) & 1 for x in [buffers[a][1]] + list(buffers[a][2]))

    for a in range(len(buffers)):
        for b in range(a + 1, len(buffers)):
            wa, wb = buffers[a][0], buffers[b][0]
            if not wa or not wb or offsets[a] + wa <= offsets[b] or offsets[b] + wb <= offsets[a]:
                continue
            assert not buffers[a][3] and not buffers[b][3], "pinned buffer %d overlaps %d" % (a if buffers[a][3] else b, b if buffers[a][3] else a)
            assert ordered(a, b) or ordered(b, a), "buffers %d and %d share words without a reader -> writer order" % (a, b)


def test_chain_reuses_two_slots():
    n, w = 10, 64
    steps = [(0, [])] * n
    buffers = [(w, i, [i + 1] if i + 1 < n else [], False) for i in range(n)]
    _, waits, peak = pack(steps, buffers)
    assert peak == 2 * w and waits == []


def test_diamond_reuses_the_source_without_a_new_wait():
    w = 32
    steps = [(0, []), (0, []), (1, [0]), (0, [2])]
    buffers = [(w, 0, [1, 2], False), (w, 1, [3], False), (w, 2, [3], False), (w, 3, [], False)]
    offsets, waits, peak = pack(steps, buffers)
    assert waits == [] and peak == 3 * w and offsets[3] == offsets[0]


def test_cross_stream_reuse_adds_one_wait():
    w = 16
    steps = [(0, []), (1, [0]), (0, []), (1, [])]
    buffers = [(w, 0, [1], False), (w, 1, [3], False), (w, 2, [], False)]
    offsets, waits, peak = pack(steps, buffers)
    assert offsets[2] == offsets[0] and peak == 2 * w
    assert waits == [(2, 1)]


def test_a_block_freed_on_the_writers_stream_is_preferred():
    w = 16
    # A read last on stream 1, B read last on stream 0; C (stream 0) takes B's words and needs no wait
    steps = [(0, []), (0, []), (1, [0]), (0, []), (0, [])]
    buffers = [(w, 0, [2], False), (w, 1, [3], False), (w, 4, [], False)]
    offsets, waits, _ = pack(steps, buffers)
    assert offsets[2] == offsets[1] and waits == []


def test_pinned_buffers_are_never_shared():
    w = 8
    steps = [(0, [])] * 6
    buffers = [(w, 0, [1], True)] + [(w, i, [i + 1], False) for i in range(1, 5)] + [(w, 5, [], True)]
    offsets, waits, peak = pack(steps, buffers)
    assert offsets[0] == 0 and offsets[-1] == w   # pinned buffers sit below the rest
    assert peak == 2 * w + 2 * w


def test_composite_buffer_lives_until_its_last_member_read():
    w = 32
    steps = [(0, [])] * 6
    # X: written at 0, one member read at 1, another at 4.  Y (2..3) cannot take X's words; Z (5) can.
    buffers = [(2 * w, 0, [1, 4], False), (w, 2, [3], False), (2 * w, 5, [], False)]
    offsets, _, peak = pack(steps, buffers)
    assert offsets[1] >= 2 * w
    assert offsets[2] == offsets[0] and peak == 3 * w


def test_no_reuse_opportunity_gives_the_sum_of_sizes():
    rng = random.Random(7)
    n = 12
    steps = [(rng.randrange(3), []) for _ in range(n)]
    steps[-1] = (0, list(range(n - 1)))
    buffers = [(rng.randrange(1, 100), i, [n - 1], False) for i in range(n - 1)]
    _, waits, peak = pack(steps, buffers)
    assert peak == sum(b[0] for b in buffers) and waits == []


def test_rejects_waits_on_later_steps():
    with pytest.raises(ValueError):
        _pack_arena([(0, [1]), (0, [])], [(8, 0, [1], False)])


def random_plan(rng):
    """a random DAG in the executor's shape: every step writes one buffer (some several-member composites read at
    different times), reads earlier ones, runs on a random stream and waits on cross-stream producers"""
    n = rng.randrange(2, 60)
    S = rng.randrange(1, 9)
    n_in = rng.randrange(0, 4)
    steps, buffers, producer = [], [], []
    for k in range(n_in):   # program inputs: pinned, uploaded before the run
        buffers.append([rng.choice([4, 8, 16]), 0, [], True])
        producer.append(None)
    for i in range(n):
        stream = rng.randrange(S)
        waits = set()
        cands = list(range(len(buffers)))
        for b in rng.sample(cands, min(len(cands), rng.randrange(0, 4))):
            buffers[b][2].append(i)
            p = producer[b]
            if p is not None and steps[p][0] != stream:
                waits.add(p)
        steps.append((stream, sorted(waits)))
        buffers.append([rng.choice([4, 8, 8, 16, 24, 64]), i, [], False])
        producer.append(i)
    for b in rng.sample(range(n_in, len(buffers)), rng.randrange(0, 3)):   # outputs and workspaces
        buffers[b][3] = True
    return steps, [tuple(b) for b in buffers]


@pytest.mark.parametrize("seed", range(300))
def test_random_dags(seed):
    rng = random.Random(seed)
    steps, buffers = random_plan(rng)
    offsets, waits, peak = pack(steps, buffers)
    assert peak <= sum(b[0] for b in buffers)
