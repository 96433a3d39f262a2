"""The ciphertext store's paging and layouts without a device: its admission is the key pager's (RegionCache::assignAll keyed
by store entry), replayed against the Python LRU model, and the byte accounting of both layouts matches shapes computed here."""
import pytest

from test_slot_cache import replay_model, replay_native


def store_batches(handles_per_batch):
    """batches of stored handles (instance order) -> batches of entry keys, numbered by first appearance: any one-to-one relabelling
    of the entries gives the same regions, fills and evictions"""
    key = {}
    return [[key.setdefault(h, len(key)) for h in batch] for batch in handles_per_batch]


def store_replay(entries, handles_per_batch):
    """(fills, evictions) of a store with `entries` device entries that resolves these batches in turn"""
    _, fills, evictions = replay_native(entries, store_batches(handles_per_batch))
    return fills, evictions


def cycling_batches(stored, per_batch, batches):
    """requests cycling over `stored` handles 1..stored, `per_batch` distinct ones per batch, each named twice"""
    out = []
    for i in range(batches):
        names = [1 + (i * per_batch + j) % stored for j in range(per_batch)]
        out.append(names + names[::-1])
    return out


def test_cycling_working_set_evicts_every_batch():
    """4 device entries, 16 stored ciphertexts named 4 at a time: every batch fills 4 entries and, once the store is warm, evicts 4"""
    batches = store_batches(cycling_batches(16, 4, 12))
    assert replay_native(4, batches) == replay_model(4, batches)
    assert store_replay(4, cycling_batches(16, 4, 12)) == (48, 44)


def test_working_set_that_fits_fills_once():
    batches = cycling_batches(4, 4, 10)
    assert store_replay(4, batches) == (4, 0)
    assert store_replay(8, cycling_batches(8, 2, 10)) == (8, 0)


def test_twice_the_entries_and_releases():
    """a working set of twice the entries, with releases (a released entry's key is dropped) in between"""
    import numpy as np
    rng = np.random.default_rng(11)
    ops = []
    for _ in range(200):
        if rng.random() < 0.1:
            ops.append(("remove", int(rng.integers(0, 16))))
        else:
            ops.append([int(x) for x in rng.integers(0, 16, int(rng.integers(1, 9)))])
    assert replay_native(8, ops) == replay_model(8, ops)


def test_too_many_distinct_entries_in_one_batch_changes_nothing():
    res, fills, evictions = replay_native(4, [[0, 1, 2, 3, 4], [0, 1]])
    assert isinstance(res[0], str) and "5 distinct" in res[0]
    assert (fills, evictions) == (2, 0)


@pytest.mark.parametrize("N,k", [(8192, 4), (16384, 7), (32768, 12)])
@pytest.mark.parametrize("storage", ["expanded", "seeded"])
def test_layout_bytes(N, k, storage):
    from eva_b200 import _eva_b200 as native
    rows = 1 if storage == "seeded" else 2
    for ell in range(1, k):
        for seeded in (False, True):
            entry, host = native._store_bytes(k, N, storage, ell, seeded)
            assert entry == rows * (k - 1) * N * 8
            assert host == (1 if seeded else 2) * ell * N * 8
    full, _ = native._store_bytes(k, N, "expanded", 1, False)
    half, _ = native._store_bytes(k, N, "seeded", 1, True)
    assert full == 2 * half


def test_layout_sobel_shape():
    """Sobel's shape (N = 16384, five primes, the image at ell = 4): a full entry is 1 MiB, a seeded one 512 KiB, on both ends"""
    from eva_b200 import _eva_b200 as native
    assert native._store_bytes(5, 16384, "expanded", 4, False) == (1 << 20, 1 << 20)
    assert native._store_bytes(5, 16384, "expanded", 4, True) == (1 << 20, 1 << 19)
    assert native._store_bytes(5, 16384, "seeded", 4, True) == (1 << 19, 1 << 19)


@pytest.mark.parametrize("bad", ["compressed", "", "Seeded"])
def test_layout_rejects_unknown_storage(bad):
    from eva_b200 import _eva_b200 as native
    with pytest.raises(ValueError, match="store_storage"):
        native._store_bytes(4, 8192, bad, 1, True)
