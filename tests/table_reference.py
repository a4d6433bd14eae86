"""The hash table's operations as plain sequential loops (reference hash_table.py:91-138 store,
:150-176 get_hits, :325-345 name_to_id, :346-383 remove / retrieve), plus the device-only
restriction to an id range and the fast matcher's pruning bound.  The device kernels of
csrc/afp_store.cu, csrc/afp_table_edit.cu and csrc/afp_match.cu are held to these by
tests/test_gpu_table_edges.py; tests/test_table_reference_cpu.py pins them to tables the
reference built and to the host mirror.

A state is any object with `hashbits`, `depth`, `maxtimebits`, `table` (uint32 [2^hashbits,
depth]), `counts` (int32 [2^hashbits]), `names` (list) and `hashesperid` (uint32) - a State or
an audfprint_b200.HashTable.  Every function changes the state in place."""
import random

import numpy as np

from oracle import afp_oracle as orc


class State(object):
    def __init__(self, hashbits, depth, maxtimebits, table=None, counts=None, names=(), hashesperid=None):
        self.hashbits, self.depth, self.maxtimebits = hashbits, depth, maxtimebits
        nb = 1 << hashbits
        self.table = np.zeros((nb, depth), np.uint32) if table is None else np.array(table, np.uint32)
        self.counts = np.zeros(nb, np.int32) if counts is None else np.array(counts, np.int32)
        self.names = list(names)
        self.hashesperid = (np.zeros(len(self.names), np.uint32) if hashesperid is None
                            else np.array(hashesperid, np.uint32))
        assert self.table.shape == (nb, depth) and self.counts.shape == (nb,)
        assert len(self.hashesperid) == len(self.names)

    def copy(self):
        return State(self.hashbits, self.depth, self.maxtimebits, self.table, self.counts, self.names,
                     self.hashesperid)


def mirror(state):
    """An audfprint_b200.HashTable holding a copy of `state`."""
    from audfprint_b200 import HashTable
    ht = HashTable(hashbits=state.hashbits, depth=state.depth, maxtime=1 << state.maxtimebits)
    ht.table, ht.counts = state.table.copy(), state.counts.copy()
    ht.names, ht.hashesperid = list(state.names), np.array(state.hashesperid, np.uint32)
    return ht


class _EveryId(object):
    """Stands in for `names` in orc.Table.store, so that its loop takes an id directly."""

    def __contains__(self, id_):
        return True

    def index(self, id_):
        return id_


def name_to_id(state, name):
    """name_to_id(name, add_if_missing=True): an int is passed through (IndexError outside the
    names), a known name keeps its id, a new one takes the first freed slot (its hashesperid
    reset to 0), else the end of the list."""
    if not isinstance(name, (str, bytes)):
        if not 0 <= int(name) < len(state.names):
            raise IndexError("track id %d outside [0, %d)" % (int(name), len(state.names)))
        return int(name)
    if name in state.names:
        return state.names.index(name)
    if None in state.names:
        i = state.names.index(None)
        state.names[i] = name
        state.hashesperid[i] = 0
        return i
    state.names.append(name)
    state.hashesperid = np.append(state.hashesperid, np.uint32(0))
    return len(state.names) - 1


def store(state, id_, rows, rng=random):
    """orc.Table.store's loop for track `id_`: row by row in call order, a bucket below `depth`
    takes the entry at slot `count`, a full one draws rng.randint(0, count) and takes it there if
    the slot is below `depth`; the count goes up by one either way."""
    if (id_ + 2) << state.maxtimebits > 1 << 32:
        raise OverflowError("id %d does not fit in %d id bits" % (id_, 32 - state.maxtimebits))
    shim = orc.Table.__new__(orc.Table)
    shim.hashbits, shim.depth, shim.maxtimebits = state.hashbits, state.depth, state.maxtimebits
    shim.table, shim.counts, shim.hashesperid, shim.names = state.table, state.counts, state.hashesperid, _EveryId()
    orc.Table.store(shim, id_, np.asarray(rows, np.int64).reshape(-1, 2).tolist(), rng)


def get_hits(state, q):
    """[id, dtime, hash, time] rows in (query row, slot) order."""
    return orc.get_hits(state.table, state.counts, state.hashbits, state.depth, state.maxtimebits, q)


def _ids(row, mtb):
    """id of every entry of a row (an empty slot gives -1)."""
    return (row >> np.uint32(mtb)).astype(np.int64) - 1


def remove(state, id_):
    """Drop every entry of track `id_`; returns how many there were.  Membership and the removed
    count are taken over the whole row; a bucket holding such an entry keeps the others among its
    first min(count, depth) slots in slot order, zero-fills the rest of the row and takes their
    number as its count.  The name becomes None and its hashesperid 0."""
    removed = 0
    for b in np.nonzero((_ids(state.table, state.maxtimebits) == id_).any(axis=1))[0]:
        row = state.table[b]
        n = min(int(state.counts[b]), state.depth)
        keep = []
        for s in range(state.depth):
            mine = (int(row[s]) >> state.maxtimebits) - 1 == id_
            removed += mine
            if s < n and not mine:
                keep.append(int(row[s]))
        row[:] = 0
        row[:len(keep)] = keep
        state.counts[b] = len(keep)
    state.names[id_] = None
    state.hashesperid[id_] = 0
    return removed


def retrieve(state, id_):
    """int32 (n, 2) [time, hash] of track `id_`'s entries among the valid slots, in (hash, slot) order."""
    tmask = (1 << state.maxtimebits) - 1
    out = []
    for b in np.nonzero((_ids(state.table, state.maxtimebits) == id_).any(axis=1))[0]:
        for s in range(min(int(state.counts[b]), state.depth)):
            v = int(state.table[b, s])
            if (v >> state.maxtimebits) - 1 == id_:
                out.append((v & tmask, int(b)))
    return np.array(out, np.int32).reshape(-1, 2)


def restrict(state, lo, hi):
    """Keep the entries of ids in [lo, hi) among every bucket's valid slots, in slot order; the
    rest of the valid slots become 0 and the count the number kept."""
    for b in np.nonzero(state.counts)[0]:
        row = state.table[b]
        n = min(int(state.counts[b]), state.depth)
        keep = [int(v) for v in row[:n] if lo <= (int(v) >> state.maxtimebits) - 1 < hi]
        row[:n] = 0
        row[:len(keep)] = keep
        state.counts[b] = len(keep)


def pruning_bound(table, counts, hashesperid, maxtimebits):
    """The smallest non-zero hashesperid; 0 if there is none, or if an entry among the valid slots
    names an id whose hashesperid is 0 (its weight would be infinite)."""
    hpi = np.asarray(hashesperid)
    nz = hpi[hpi != 0]
    if len(nz) == 0:
        return 0
    zero = set(np.nonzero(hpi == 0)[0].tolist())
    if zero:
        depth = table.shape[1]
        for b in np.nonzero(counts)[0]:
            for v in table[b, :min(int(counts[b]), depth)]:
                if (int(v) >> maxtimebits) - 1 in zero:
                    return 0
    return int(nz.min())
