"""The host restatement of the device node tables (tests/hash_layout.py), checked without a GPU:
  * probe_pos visits every slot once from any home;
  * on hand-built tables of adversarial key sets (long chains, chains that wrap past the last slot, interleaved buddy
    chains, misses that walk a foreign chain) probe_slot and both halves of the sector walk equal a Python dict;
  * the invariant checker accepts every such table, whatever the insertion order, and rejects three corruptions the
    sector walk cannot survive: a maxdisp2 lowered by one, a hole punched in a chain and a wrong key2."""
import numpy as np
import pytest

from tests import hash_layout as hl

CAPS = [64, 256, 4096]


def _table(cap, seed, level=8, load=0.85, shuffle=False):
    rng = np.random.default_rng(seed)
    ks = hl.adversarial_keys(rng, cap, level, load)
    keys = ks["stored"]
    ids = rng.integers(0, 10 ** 6, size=(keys.size, 8)).astype(np.int32)
    order = rng.permutation(keys.size) if shuffle else np.arange(keys.size)
    s = hl.Slots(cap)
    for i in order:
        s.insert(int(keys[i]), int(i), ids[i])
    return s, ks, keys, ids


def test_hash_key_matches_known_values():
    # the device mix on a few keys, computed by hand with Python integers
    def ref(k):
        m = (1 << 64) - 1
        k ^= k >> 31; k = (k * 0x9E3779B97F4A7C15) & m
        k ^= k >> 29; k = (k * 0xBF58476D1CE4E5B9) & m
        k ^= k >> 32
        return k & 0xFFFFFFFF
    keys = [0, 1, 7, 8 ** 12 - 1, 0x123456789A, 2 ** 47 + 3]
    assert hl.hash_key(np.array(keys, dtype=np.int64)).tolist() == [ref(k) for k in keys]


@pytest.mark.parametrize("cap", [2, 16, 64])
def test_probe_sequence_visits_every_slot_once(cap):
    for h0 in range(cap):
        seq = hl.probe_pos(np.full(cap, h0), np.arange(cap), cap - 1)
        assert sorted(seq.tolist()) == list(range(cap))
        assert np.array_equal(hl.probe_index(np.full(cap, h0), seq, cap - 1), np.arange(cap))


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("shuffle", [False, True])
def test_walks_equal_a_dict(cap, shuffle):
    s, ks, keys, ids = _table(cap, cap + shuffle, shuffle=shuffle)
    d = {int(k): ids[i] for i, k in enumerate(keys)}
    rng = np.random.default_rng(cap)
    probes = np.concatenate((keys, ks["absent_chain"], ks["absent"], rng.integers(0, 8 ** 8, size=200)))
    for k in probes.tolist():
        want = d.get(k)
        for half in (None, 0, 1):
            got = hl.lookup(s, k, half)
            if want is None:
                assert got is None, (k, half)
            elif half is None:
                assert np.array_equal(got, want), (k, half)
            else:
                assert np.array_equal(got, want[half::2]), (k, half)
    info = hl.check_slots(s, keys, ids)
    # the key sets really are adversarial
    hc, hb, last = ks["homes"]
    mask = cap - 1
    it = [hl.probe_index(hl.hash_key(k) & mask, hl.probe_slot(s, k), mask) for k in ks["cluster"]]
    assert max(it) >= 7, it                                               # 8 keys of one home: a chain of 8 probes
    wrapped = [hl.probe_slot(s, k) for k in ks["wrap"]]
    assert min(wrapped) < last - 1, wrapped                               # past the last slot, on to slot 0 ...
    for k in ks["absent_chain"]:                                          # misses that walk a foreign chain
        h0 = int(hl.hash_key(k)) & mask
        assert s.key[h0] != hl.EMPTY and s.key[h0] != np.uint64(k) and s.maxdisp[h0] > 1
    print(f"cap {cap}: {info}")


def _far_key(s, keys):
    """(index in keys, home, probe index) of a key that sits at probe >= 2 and is the farthest key of its home."""
    mask = s.mask
    for i, k in enumerate(keys.tolist()):
        h0 = int(hl.hash_key(k)) & mask
        slot = hl.probe_slot(s, k)
        it = int(hl.probe_index(h0, slot, mask))
        if it >= 2 and it == s.maxdisp[h0]:
            return i, h0, it
    raise AssertionError("no key at probe >= 2")


@pytest.mark.parametrize("cap", CAPS)
def test_checker_rejects_a_lowered_maxdisp2(cap):
    s, _, keys, ids = _table(cap, 7)
    i, h0, it = _far_key(s, keys)
    bad = s.copy()
    bad.maxdisp2[h0] -= 1
    with pytest.raises(AssertionError, match="maxdisp2"):
        hl.check_slots(bad, keys, ids)
    assert hl.lookup(bad, keys[i], 1) is None and hl.lookup(bad, keys[i], 0) is not None   # the sector-1 lane misses


@pytest.mark.parametrize("cap", CAPS)
def test_checker_rejects_a_hole_in_a_chain(cap):
    s, _, keys, ids = _table(cap, 8)
    i, h0, it = _far_key(s, keys)
    hole = int(hl.probe_pos(h0, it - 1, s.mask))                         # the slot just before the key on its walk
    r = int(s.node[hole])
    bad = s.copy()
    bad.key[hole] = bad.key2[hole] = hl.EMPTY
    bad.node[hole], bad.ids0[hole], bad.ids1[hole] = -1, -1, -1
    bad.node[bad.node > r] -= 1                                          # the table of the keys without keys[r]
    keep = np.arange(keys.size) != r
    with pytest.raises(AssertionError, match="free slot on the walk"):
        hl.check_slots(bad, keys[keep], ids[keep])
    assert all(hl.lookup(bad, keys[i], half) is None for half in (None, 0, 1))   # the walk stops at the hole


@pytest.mark.parametrize("cap", CAPS)
def test_checker_rejects_a_wrong_key2(cap):
    s, _, keys, ids = _table(cap, 9)
    i, h0, it = _far_key(s, keys)
    bad = s.copy()
    bad.key2[h0] = np.uint64(int(keys[i]))                               # the home's copy names the displaced key
    with pytest.raises(AssertionError, match="key2"):
        hl.check_slots(bad, keys, ids)
    assert not np.array_equal(hl.lookup(bad, keys[i], 1), hl.lookup(s, keys[i], 1))   # the home's rows, not the key's


def test_encode_decode_round_trip():
    s, _, keys, ids = _table(256, 10)
    raw = s.encode()
    assert raw.size == 256 * hl.SLOT_BYTES
    back = hl.Slots.decode(raw)
    for name in ("key", "key2", "node", "pad1", "maxdisp", "maxdisp2", "ids0", "ids1"):
        assert np.array_equal(getattr(back, name), getattr(s, name)), name
    free = hl.Slots(64).encode()
    assert np.all(free == 0xFF)                                          # a free slot is all 0xFF bytes
