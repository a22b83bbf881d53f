"""Host restatement of the device node tables (csrc/shine_device.cuh): the 64-byte `HashSlot`, `hash_key`, `probe_pos`,
the two walks that read them (`probe_slot`, and `resolve_sector` for each 32-byte half), the invariants every build path
must leave behind, and key sets that make the walks work hard.  Test infrastructure, no GPU needed.

Slot layout (bytes): key 0-7 | node 8-11 | maxdisp 12-15 | ids0 16-31 (corners 0 2 4 6) | key2 32-39 | pad1 40-43 |
maxdisp2 44-47 | ids1 48-63 (corners 1 3 5 7).  A free slot is all 0xFF bytes (key = EMPTY, maxdisp = maxdisp2 = -1).

Invariants (`check_slots`), for every stored key at probe index `it` of its home h0:
  * key2 == key;
  * it <= maxdisp[h0] == maxdisp2[h0] (a walk from h0 never stops before the key, in either half);
  * no free slot at probe indices < it (a walk stops at the first free slot);
  * node and the 8 corner rows equal node_keys / node_ids at that node's index.
"""
from __future__ import annotations

import numpy as np

EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
SLOT_BYTES = 64


def hash_key(k) -> np.ndarray:
    """hash_key of shine_device.cuh in uint64 arithmetic (wraps like the device's) -> int64 in [0, 2^32)."""
    k = np.asarray(k).astype(np.uint64)
    with np.errstate(over="ignore"):
        k = k ^ (k >> np.uint64(31))
        k = k * np.uint64(0x9E3779B97F4A7C15)
        k = k ^ (k >> np.uint64(29))
        k = k * np.uint64(0xBF58476D1CE4E5B9)
        k = k ^ (k >> np.uint64(32))
    return (k & np.uint64(0xFFFFFFFF)).astype(np.int64)


def probe_pos(h0, it, mask):
    """probe_pos of shine_device.cuh, vectorised over h0 / it: h0, its buddy h0 ^ 1, then linearly from the next pair."""
    h0, it = np.asarray(h0), np.asarray(it)
    return np.where(it == 0, h0, np.where(it == 1, h0 ^ 1, ((h0 & ~1) + it) & mask))


def probe_index(h0, s, mask):
    """Inverse of probe_pos: the probe index at which a key of home h0 sits in slot s."""
    h0, s = np.asarray(h0), np.asarray(s)
    return np.where(s == h0, 0, np.where(s == (h0 ^ 1), 1, (s - (h0 & ~1)) & mask))


class Slots:
    """A node table as host arrays, decoded from (or encodable to) the raw 64-byte slots."""

    def __init__(self, capacity: int):
        assert capacity >= 2 and capacity & (capacity - 1) == 0
        self.capacity = capacity
        self.key = np.full(capacity, EMPTY, dtype=np.uint64)
        self.key2 = np.full(capacity, EMPTY, dtype=np.uint64)
        self.node = np.full(capacity, -1, dtype=np.int32)
        self.pad1 = np.full(capacity, -1, dtype=np.int32)
        self.maxdisp = np.full(capacity, -1, dtype=np.int32)
        self.maxdisp2 = np.full(capacity, -1, dtype=np.int32)
        self.ids0 = np.full((capacity, 4), -1, dtype=np.int32)
        self.ids1 = np.full((capacity, 4), -1, dtype=np.int32)

    @property
    def mask(self) -> int:
        return self.capacity - 1

    @classmethod
    def decode(cls, raw) -> "Slots":
        raw = np.ascontiguousarray(np.asarray(raw, dtype=np.uint8)).reshape(-1, SLOT_BYTES)
        s = cls(raw.shape[0])
        s.key = raw[:, 0:8].copy().view(np.uint64)[:, 0]
        s.node = raw[:, 8:12].copy().view(np.int32)[:, 0]
        s.maxdisp = raw[:, 12:16].copy().view(np.int32)[:, 0]
        s.ids0 = raw[:, 16:32].copy().view(np.int32)
        s.key2 = raw[:, 32:40].copy().view(np.uint64)[:, 0]
        s.pad1 = raw[:, 40:44].copy().view(np.int32)[:, 0]
        s.maxdisp2 = raw[:, 44:48].copy().view(np.int32)[:, 0]
        s.ids1 = raw[:, 48:64].copy().view(np.int32)
        return s

    def encode(self) -> np.ndarray:
        raw = np.empty((self.capacity, SLOT_BYTES), dtype=np.uint8)
        for lo, a in ((0, self.key), (8, self.node), (12, self.maxdisp), (16, self.ids0), (32, self.key2),
                      (40, self.pad1), (44, self.maxdisp2), (48, self.ids1)):
            b = np.ascontiguousarray(a).view(np.uint8).reshape(self.capacity, -1)
            raw[:, lo:lo + b.shape[1]] = b
        return raw.reshape(-1)

    def copy(self) -> "Slots":
        out = Slots(self.capacity)
        out.__dict__.update({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in self.__dict__.items()})
        return out

    def insert(self, key: int, node: int, ids) -> int:
        """hash_insert_kernel for one key, sequentially: the first free (or equal) slot on the key's walk -> slot."""
        key = np.uint64(key)
        h0 = int(hash_key(key))
        h0 &= self.mask
        for it in range(self.capacity):
            h = int(probe_pos(h0, it, self.mask))
            if self.key[h] == EMPTY or self.key[h] == key:
                self.key[h] = self.key2[h] = key
                self.node[h] = node
                ids = np.asarray(ids, dtype=np.int32)
                self.ids0[h], self.ids1[h] = ids[0::2], ids[1::2]
                if it > 0:
                    self.maxdisp[h0] = max(self.maxdisp[h0], it)
                    self.maxdisp2[h0] = max(self.maxdisp2[h0], it)
                return h
        raise OverflowError("table full")


def build(capacity: int, keys, ids=None) -> Slots:
    """A table holding `keys` in this order, node i = keys[i], corner rows ids[i] (default 8 i .. 8 i + 7)."""
    keys = np.asarray(keys, dtype=np.int64)
    ids = np.arange(8 * keys.size, dtype=np.int32).reshape(-1, 8) if ids is None else np.asarray(ids, dtype=np.int32)
    s = Slots(capacity)
    for i, k in enumerate(keys):
        s.insert(int(k), i, ids[i])
    return s


def _walk(s: Slots, h0: int, key: np.uint64, last: int) -> int:
    """probe_slot_from: probes 1 .. last of home h0, reading each slot's sector-0 key; stops at a free slot."""
    for n in range(1, last + 1):
        h = int(probe_pos(h0, n, s.mask))
        if s.key[h] == key:
            return h
        if s.key[h] == EMPTY:
            return -1
    return -1


def probe_slot(s: Slots, key: int) -> int:
    """probe_slot of shine_device.cuh: the home slot's sector 0 (key, maxdisp) bounds the walk -> slot or -1."""
    key = np.uint64(key)
    h0 = int(hash_key(key)) & s.mask
    if s.key[h0] == key:
        return h0
    if s.key[h0] == EMPTY or s.maxdisp[h0] <= 0:
        return -1
    return _walk(s, h0, key, int(s.maxdisp[h0]))


def resolve_sector(s: Slots, key: int, half: int):
    """The sector walk of one lane: sector `half` of the home slot (key / maxdisp, or key2 / maxdisp2), then the
    continuation over sector-0 keys -> (slot or -1, the lane's 4 corner rows or -1 x 4)."""
    key = np.uint64(key)
    h0 = int(hash_key(key)) & s.mask
    k, md = (s.key[h0], s.maxdisp[h0]) if half == 0 else (s.key2[h0], s.maxdisp2[h0])
    ids = s.ids0 if half == 0 else s.ids1
    if k == key:
        return h0, ids[h0].copy()
    slot = _walk(s, h0, key, int(md)) if (k != EMPTY and md > 0) else -1
    return slot, (ids[slot].copy() if slot >= 0 else np.full(4, -1, dtype=np.int32))


def lookup(s: Slots, key: int, half: int | None = None):
    """The 8 corner rows a walk yields (half None: probe_slot; 0 / 1: both lanes' sector walks) or None on a miss.  The
    two lanes of the sector walk must agree on hit / miss."""
    if half is None:
        slot = probe_slot(s, key)
        if slot < 0:
            return None
        out = np.empty(8, dtype=np.int32)
        out[0::2], out[1::2] = s.ids0[slot], s.ids1[slot]
        return out
    slot, ids = resolve_sector(s, key, half)
    return None if slot < 0 else ids


def check_slots(s: Slots, node_keys, node_ids, what="table"):
    """Assert the invariants of the module docstring for a table that must hold exactly node_keys (node i = node_keys[i],
    its corner rows node_ids[i])."""
    node_keys = np.asarray(node_keys, dtype=np.int64)
    node_ids = np.asarray(node_ids, dtype=np.int32).reshape(-1, 8)
    n, mask = node_keys.size, s.mask
    assert np.unique(node_keys).size == n, f"{what}: node_keys has duplicates"
    occupied = np.flatnonzero(s.key != EMPTY)
    assert occupied.size == n, f"{what}: {occupied.size} occupied slots for {n} nodes"
    assert n < s.capacity, f"{what}: no free slot left"
    bad = occupied[s.key2[occupied] != s.key[occupied]]
    assert bad.size == 0, f"{what}: key2 != key in slot {bad[0]}"
    slot_keys = s.key[occupied].astype(np.int64)
    order = np.argsort(slot_keys)
    assert np.array_equal(slot_keys[order], np.sort(node_keys)), f"{what}: slot keys != node_keys"
    slot = np.empty(n, dtype=np.int64)
    slot[np.argsort(node_keys)] = occupied[order]                      # slot of node i
    assert np.array_equal(s.node[slot], np.arange(n)), f"{what}: slot ordinal != index in node_keys"
    assert np.array_equal(s.ids0[slot], node_ids[:, 0::2]), f"{what}: ids0 != node_ids (even corners)"
    assert np.array_equal(s.ids1[slot], node_ids[:, 1::2]), f"{what}: ids1 != node_ids (odd corners)"
    h0 = hash_key(node_keys) & mask
    it = probe_index(h0, slot, mask)
    far = it > 0
    j = np.flatnonzero(far & (it > s.maxdisp[h0]))
    assert j.size == 0, f"{what}: key {node_keys[j[0]]} at probe {it[j[0]]} beyond its home's maxdisp {s.maxdisp[h0[j[0]]]}"
    j = np.flatnonzero(far & (it > s.maxdisp2[h0]))
    assert j.size == 0, f"{what}: key {node_keys[j[0]]} at probe {it[j[0]]} beyond its home's maxdisp2 {s.maxdisp2[h0[j[0]]]}"
    for jj in np.flatnonzero(far):                                     # no free slot before the key on its walk
        walk = probe_pos(np.full(it[jj], h0[jj]), np.arange(it[jj]), mask)
        assert np.all(s.key[walk] != EMPTY), f"{what}: free slot on the walk of key {node_keys[jj]} before probe {it[jj]}"
    d = np.flatnonzero(s.maxdisp != s.maxdisp2)
    assert d.size == 0, f"{what}: maxdisp {s.maxdisp[d[0]]} != maxdisp2 {s.maxdisp2[d[0]]} at slot {d[0]}"
    # every home: maxdisp == maxdisp2 == the largest probe index of its displaced keys (<= 0 when none was displaced)
    want = np.full(s.capacity, -1, dtype=np.int64)
    np.maximum.at(want, h0[far], it[far])
    got = np.maximum(s.maxdisp.astype(np.int64), -1)
    got2 = np.maximum(s.maxdisp2.astype(np.int64), -1)
    d = np.flatnonzero((np.maximum(got, 0) != np.maximum(want, 0)) | (np.maximum(got2, 0) != np.maximum(want, 0)))
    assert d.size == 0, (f"{what}: home {d[0]} has maxdisp {s.maxdisp[d[0]]} / maxdisp2 {s.maxdisp2[d[0]]}, its farthest "
                         f"key sits at probe {max(int(want[d[0]]), 0)}")
    return {"nodes": n, "capacity": s.capacity, "max_probe": int(it.max()) if n else 0}


# ---- adversarial key sets ------------------------------------------------------------------------------------------------

def keys_with_home(rng, capacity: int, level: int, homes, per_home: int, exclude=()):
    """per_home distinct Morton codes of `level` whose home slot is each of `homes` (in homes order) -> int64 [len * per]."""
    mask = capacity - 1
    homes = np.asarray(homes, dtype=np.int64)
    taken = set(int(k) for k in exclude)
    found = {int(h): [] for h in homes}
    hi = 8 ** level
    while any(len(v) < per_home for v in found.values()):
        cand = rng.integers(0, hi, size=max(1 << 18, 64 * capacity), dtype=np.int64)
        hh = hash_key(cand) & mask
        for h in found:
            if len(found[h]) >= per_home:
                continue
            for k in cand[hh == h].tolist():
                if k not in taken and len(found[h]) < per_home:
                    taken.add(k)
                    found[h].append(k)
    return np.array([k for h in homes for k in found[int(h)]], dtype=np.int64)


def adversarial_keys(rng, capacity: int, level: int, load: float = 0.85, include=()):
    """Stored and absent Morton codes of `level` for a table of `capacity` slots:
      * `cluster`: 8 keys with one home (a chain through the buddy slot and 6 linear probes);
      * `wrap`: 5 keys homed at the last slot and 3 at the one before (their chains wrap past the end to slot 0);
      * `buddy`: 4 keys homed at an even slot h and 4 at h + 1 (the two chains interleave);
      * filler keys at random homes up to `load` (chains of different homes merge);
      * `absent_chain`: keys not stored whose home is the cluster's or the last slot (a different key, maxdisp > 1: the
        miss walks the whole chain), `absent`: random keys not stored.
    include: keys that must be stored too (inserted first).
    -> dict of int64 arrays; `stored` is the insertion order (include, then the named groups)."""
    assert capacity >= 64
    mask = capacity - 1
    include = np.asarray(include, dtype=np.int64)
    hc = int(rng.integers(8, capacity // 2)) & ~1
    hb = (hc + capacity // 4) & mask & ~1
    cluster = keys_with_home(rng, capacity, level, [hc], 8, include)
    wrap = keys_with_home(rng, capacity, level, [mask], 5, np.concatenate((include, cluster)))
    wrap = np.concatenate((wrap, keys_with_home(rng, capacity, level, [mask - 1], 3,
                                                np.concatenate((include, cluster, wrap)))))
    named = np.concatenate((include, cluster, wrap))
    buddy = keys_with_home(rng, capacity, level, [hb, hb + 1], 4, named)
    named = np.concatenate((named, buddy))
    absent_chain = keys_with_home(rng, capacity, level, [hc, mask], 3, named)
    n_fill = max(0, int(load * capacity) - named.size)
    taken = set(named.tolist()) | set(absent_chain.tolist())
    fill = []
    while len(fill) < n_fill:
        for k in rng.integers(0, 8 ** level, size=2 * n_fill, dtype=np.int64).tolist():
            if k not in taken and len(fill) < n_fill:
                taken.add(k)
                fill.append(k)
    absent = []
    while len(absent) < 64:
        k = int(rng.integers(0, 8 ** level))
        if k not in taken:
            taken.add(k)
            absent.append(k)
    stored = np.concatenate((named, np.array(fill, dtype=np.int64)))
    return {"stored": stored, "cluster": cluster, "wrap": wrap, "buddy": buddy, "absent_chain": absent_chain,
            "absent": np.array(absent, dtype=np.int64), "homes": (hc, hb, mask)}
