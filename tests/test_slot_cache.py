"""The key pager's residency policy (eva_b200/csrc/host/slot_cache.hpp) against a small Python LRU model: the same slots, fills,
evictions and errors on seeded random batch sequences.  Host only."""
import numpy as np
import pytest


class LruModel:
    """every distinct tenant of a batch is pinned; a missing tenant (in order of first appearance) takes the lowest free slot, else
    the least recently used slot no tenant of the batch holds"""

    def __init__(self, slots):
        self.S = slots
        self.owner, self.stamp, self.slot = [-1] * slots, [0] * slots, {}
        self.clock = self.fills = self.evictions = 0

    def assign(self, tenants):
        distinct = list(dict.fromkeys(tenants))
        if len(distinct) > self.S:
            return "a batch names %d distinct tenants but the key bank has %d device slots" % (len(distinct), self.S)
        pinned = {self.slot[t] for t in distinct if t in self.slot}
        fills = []
        for t in distinct:
            if t not in self.slot:
                free = [s for s in range(self.S) if self.owner[s] < 0]
                s = free[0] if free else min((s for s in range(self.S) if s not in pinned), key=lambda s: self.stamp[s])
                old = self.owner[s]
                if old >= 0:
                    del self.slot[old]
                    self.evictions += 1
                self.owner[s], self.slot[t] = t, s
                pinned.add(s)
                fills.append((t, s, old))
                self.fills += 1
            self.clock += 1
            self.stamp[self.slot[t]] = self.clock
        return ([self.slot[t] for t in tenants], fills)

    def drop(self, t):
        if t in self.slot:
            s = self.slot.pop(t)
            self.owner[s], self.stamp[s] = -1, 0


def replay_model(slots, ops):
    m = LruModel(slots)
    out = []
    for op in ops:
        if isinstance(op, tuple):
            m.drop(op[1])
            out.append(None)
        else:
            r = m.assign(op)
            out.append(r if isinstance(r, str) else (r[0], r[1]))
    return out, m.fills, m.evictions


def replay_native(slots, ops):
    from eva_b200 import _eva_b200 as native
    res, fills, ev = native._slot_cache(slots, ops)
    norm = []
    for r in res:
        if r is None or isinstance(r, str):
            norm.append(r)
        else:
            norm.append((list(r[0]), [tuple(f) for f in r[1]]))
    return norm, fills, ev


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("slots", [1, 2, 3, 5, 8])
def test_slot_cache_matches_lru_model(seed, slots):
    rng = np.random.default_rng(1000 * slots + seed)
    ops = []
    for _ in range(60):
        if rng.random() < 0.08:
            ops.append(("remove", int(rng.integers(0, 12))))
        else:
            n = int(rng.integers(1, 2 * slots + 2))
            hot = int(rng.integers(slots, 13))          # tenants drawn from a window: hits, misses and too-many errors
            ops.append([int(t) for t in rng.integers(0, hot, n)])
    assert replay_native(slots, ops) == replay_model(slots, ops)


def test_slot_cache_pins_the_batch_and_evicts_lru():
    res, fills, ev = replay_native(2, [[0], [1], [0], [2], [1, 2], [0, 2, 0], [0, 1, 2]])
    assert res[0] == ([0], [(0, 0, -1)]) and res[1] == ([1], [(1, 1, -1)])
    assert res[2] == ([0], [])                       # hit: 0 becomes the most recent
    assert res[3] == ([1], [(2, 1, 1)])              # 1 is the least recently used
    assert res[4] == ([0, 1], [(1, 0, 0)])           # 2 is pinned by the batch: 1 takes 0's slot although 2 is older
    assert res[5] == ([0, 1, 0], [(0, 0, 1)])        # 2 pinned again: 0 takes the other slot, 1's; a repeated tenant fills once
    assert res[6] == "a batch names 3 distinct tenants but the key bank has 2 device slots"
    assert (fills, ev) == (5, 3)
