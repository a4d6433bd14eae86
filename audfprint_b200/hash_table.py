"""HashTable — drop-in mirror of hash_table.HashTable with a device-resident
copy of the bucket arrays for probing (hash_table.py:49-391).

The public attributes the reference's callers read directly (`table`, `counts`,
`names`, `hashesperid`, `params`, `hashbits`, `depth`, `maxtimebits`, `dirty`,
`ht_version`) are plain host NumPy arrays / Python objects and remain the
source of truth; `get_hits` (the hot method, 92 % of the reference's match
time) runs on the GPU against a lazily refreshed device copy.  `store` exists
twice: per track on the host, and batched on the device (`store_batch`,
SURVEY.md §8f-1: the device copy then leads and the host arrays refresh from it
when read).  `remove` and `retrieve` also exist batched on the device (`remove_batch`,
`retrieve_batch`), which the per-name forms use while the device copy leads; `merge` is
host bookkeeping.  All of them reproduce the
reference's results exactly, including its draws from the global `random` /
`np.random` generators on bucket overflow.
"""
from __future__ import annotations

import ctypes as C
import gzip
import io
import itertools
import math
import os
import pickle
import random
import sys
import weakref

import numpy as np

from . import _lib

HT_VERSION = 20170724
HT_COMPAT_VERSION = 20170724
HT_OLD_COMPAT_VERSION = 20140920


class AfpStateError(RuntimeError):
    pass


def _bitsfor(maxval):
    """log2 of a power of two, ValueError otherwise (hash_table.py:40-46)."""
    bits = int(round(math.log(maxval) / math.log(2)))
    if maxval != (1 << bits):
        raise ValueError("maxval must be a power of 2, not %d" % maxval)
    return bits


class _RefUnpickler(pickle.Unpickler):
    """Reads databases pickled by the reference (class path hash_table.HashTable)."""

    def find_class(self, module, name):
        if name == "HashTable" and module in ("hash_table", "audfprint.hash_table", __name__):
            return HashTable
        return super().find_class(module, name)


_REF_ATTRS = ("hashbits", "depth", "maxtimebits", "table", "counts", "names", "hashesperid", "params",
              "ht_version", "dirty")


class _reference_pickle_class(object):
    """Context manager yielding a class that pickles as `hash_table.HashTable`.
    pickle stores only the class PATH and checks at dump time that the path resolves to the very
    class being pickled, so a stand-in module of that name holds a stand-in class for the
    duration of the dump; whatever `hash_table` was before (nothing, the reference's module, or
    this module under that name - INTEGRATION.md option A) is put back afterwards."""
    _missing = object()

    def __enter__(self):
        import sys
        import types
        mod = types.ModuleType("hash_table")
        cls = type("HashTable", (object,), {"__module__": "hash_table"})
        mod.HashTable = cls
        self._prev = sys.modules.get("hash_table", self._missing)
        sys.modules["hash_table"] = mod
        return cls

    def __exit__(self, *exc):
        import sys
        if self._prev is self._missing:
            sys.modules.pop("hash_table", None)
        else:
            sys.modules["hash_table"] = self._prev
        return False


def _as_reference_object(ht, cls):
    """An instance of `cls` (see _reference_pickle_class) carrying exactly the reference's
    attribute set."""
    obj = object.__new__(cls)
    obj.__dict__.update({k: getattr(ht, k) for k in _REF_ATTRS})
    obj.__dict__["dirty"] = False
    return obj


class HashTable(object):
    """Fixed-array hash table of (id, time) entries keyed by landmark hash."""

    def __init__(self, filename=None, hashbits=20, depth=100, maxtime=16384, device=None):
        self.device = device
        self._init_device_state()
        if filename is not None:
            self.load(filename)
            return
        # empty table of 2^hashbits buckets x depth slots (hash_table.py:60-81)
        self.hashbits, self.depth, self.maxtimebits = hashbits, depth, _bitsfor(maxtime)
        self.table = np.zeros((1 << hashbits, depth), dtype=np.uint32)
        self.counts = np.zeros(1 << hashbits, dtype=np.int32)
        self.names, self.hashesperid = [], np.zeros(0, np.uint32)
        self.params, self.ht_version, self.dirty = {}, HT_VERSION, True

    # ---- host arrays <-> device copy bookkeeping ------------------------------------
    # `table`, `counts` and `hashesperid` are the reference's public attributes
    # (hash_table.py:59-81).  They are properties here so that (a) REBINDING one of them
    # (`ht.table = other`) is seen by the device copy, and (b) after a device-side
    # `store_batch` the host arrays are refreshed from the device before anyone reads them.
    # Writing INTO the arrays in place (`ht.table[b, s] = v`) cannot be observed: call
    # `ht.touch()` afterwards (every mutating method of this class does).
    _tokens = itertools.count(1)

    def _init_device_state(self):
        self._token = next(HashTable._tokens)   # process-unique: never equal to another table's
        self._version = 0                       # bumped on every change of the host state
        self._dev_newer = False                 # device copy holds inserts the host arrays lack
        self._shard = None

    def _bump(self):
        self._version = getattr(self, "_version", 0) + 1

    def touch(self):
        """Tell the device copy that the host arrays were modified in place."""
        self._bump()

    def _host(self, attr):
        if getattr(self, "_dev_newer", False):
            self._pull_device()
        return self.__dict__[attr]

    table = property(lambda self: self._host("_table"),
                     lambda self, a: (self.__dict__.__setitem__("_table", a), self._bump())[0])
    counts = property(lambda self: self._host("_counts"),
                      lambda self, a: (self.__dict__.__setitem__("_counts", a), self._bump())[0])
    hashesperid = property(lambda self: self.__dict__["_hashesperid"],
                           lambda self, a: (self.__dict__.__setitem__("_hashesperid", a), self._bump())[0])

    # ---- pickling: only plain host state travels (reference pickles the object) ----
    def __getstate__(self):
        if getattr(self, "_dev_newer", False):
            self._pull_device()
        st = dict(self.__dict__)
        for k in ("_token", "_version", "_dev_newer", "_shard", "_dev_key", "_store_pending"):
            st.pop(k, None)
        for k in ("table", "counts", "hashesperid"):      # the reference's attribute names
            st[k] = st.pop("_" + k)
        return st

    def __setstate__(self, st):
        st = dict(st)
        st.pop("_dev_stamp", None)
        for k in ("table", "counts", "hashesperid"):
            if k in st:
                st["_" + k] = st.pop(k)
        self.__dict__.update(st)
        self.__dict__.setdefault("device", None)
        self._init_device_state()

    def _touch(self):
        self._bump()
        self.dirty = True

    def reset(self):
        """Empty the table, keep the geometry (hash_table.py:83-89)."""
        self.table.fill(0)
        self.counts.fill(0)
        self.names, self.hashesperid = [], np.zeros(0, np.uint32)
        self._touch()

    # ---- mutation (host) ---------------------------------------------------------
    def store(self, name, timehashpairs):
        """Insert (time, hash) pairs under `name` (hash_table.py:91-138).

        Same sequential semantics as the reference, evaluated in two parts: rows
        that land below `depth` are written with one vectorised scatter; rows
        that hit a full bucket are replayed one by one, drawing
        random.randint(0, count) in the original order, so a table built here
        equals one built by the reference from the same RNG state."""
        id_ = self.name_to_id(name, add_if_missing=True)
        pairs = np.asarray(timehashpairs, dtype=np.int64).reshape(-1, 2)
        n = pairs.shape[0]
        if n:
            hmask = (1 << self.hashbits) - 1
            tmask = (1 << self.maxtimebits) - 1
            if (id_ + 2) << self.maxtimebits > (1 << 32):
                raise OverflowError("id %d does not fit in %d id bits" % (id_, 32 - self.maxtimebits))
            h = pairs[:, 1] & hmask
            vals = (((id_ + 1) << self.maxtimebits) + (pairs[:, 0] & tmask)).astype(np.uint32)
            # occurrence index of every row among equal hashes, in call order
            order = np.argsort(h, kind="stable")
            hs = h[order]
            first = np.r_[True, hs[1:] != hs[:-1]]
            grp_start = np.maximum.accumulate(np.where(first, np.arange(n), 0))
            occ = np.empty(n, np.int64)
            occ[order] = np.arange(n) - grp_start
            pos = self.counts[h].astype(np.int64) + occ
            direct = pos < self.depth
            self.table[h[direct], pos[direct]] = vals[direct]
            for i in np.nonzero(~direct)[0]:
                slot = random.randint(0, int(pos[i]))
                if slot < self.depth:
                    self.table[h[i], slot] = vals[i]
            np.add.at(self.counts, h, 1)
        self.hashesperid[id_] += n
        self._touch()

    # ---- batched insert on the device table (SURVEY.md §8f-1) ------------------------------
    def store_batch(self, names, hashes=None):
        """HashTable.store (hash_table.py:91-138) for a list of tracks in ONE device call.

        names   track names, in insertion order
        hashes  list of (time, hash) arrays, one per name - or None: the tracks are the files of the
                last Analyzer device batch and their hashes are taken from the device workspace
                without a round trip (Analyzer.ingest_batch)
        The result is the table the reference builds by calling store() track by track from the
        same `random` state: slots below `depth` are assigned on the device (rank of every entry
        inside its bucket, in insertion order); entries that meet a full bucket come back in
        order, `random.randint(0, count)` is replayed for them on a C copy of CPython's generator
        (and `random`'s state advanced accordingly), and the winning writes return as patches.
        Afterwards the DEVICE copy is the current one; `table` / `counts` refresh themselves from
        it when read.  Returns the number of hashes stored per track."""
        return self.store_batch_finish(self.store_batch_begin(names, hashes))

    def store_batch_begin(self, names, hashes=None):
        """First half of store_batch: everything up to and including the device kernels (slots
        below `depth` written, overflow entries compacted, their counts fetched).  The returned
        token goes to store_batch_finish, which replays `random.randint` for the overflow on the
        host and applies the result.  Analyzer.ingest_batch launches the NEXT batch's fingerprint
        kernels between the two, so the (sequential, host-side) RNG replay of batch k runs while the
        GPU fingerprints batch k+1; finishes must be called in the order of the begins, each
        before the next begin."""
        nfiles = len(names)
        if nfiles == 0:
            return None
        if self._shard is not None:
            raise AfpStateError("the device copy is a shard (restrict_device_ids): cannot store into it")
        if getattr(self, "_store_pending", False):
            raise AfpStateError("store_batch_begin: the previous batch was not finished")
        ctx = self._sync_device()                 # the device holds this table's current state
        ids = self._names_to_ids(names)           # (host bookkeeping; the device copy stays the current one)
        nov = C.c_int64(0)
        if hashes is None:
            roff = np.empty(nfiles + 1, np.int64)
            ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, None, 1, roff.ctypes.data_as(C.POINTER(C.c_int64))))
            ctx.check(ctx.lib.afp_table_store_batch(ctx.h, None, 0, None, nfiles, ids.ctypes.data_as(C.POINTER(C.c_int64)),
                                                    C.byref(nov)))
        else:
            arrs = [np.asarray(h, dtype=np.int32).reshape(-1, 2) for h in hashes]
            roff = np.zeros(nfiles + 1, np.int64)
            roff[1:] = np.cumsum([len(a) for a in arrs])
            rows = np.ascontiguousarray(np.concatenate(arrs)) if roff[-1] else np.zeros((0, 2), np.int32)
            ctx.check(ctx.lib.afp_table_store_batch(ctx.h, rows.ctypes.data if len(rows) else None, 1,
                                                    roff.ctypes.data_as(C.POINTER(C.c_int64)), nfiles,
                                                    ids.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(nov)))
        n = int(nov.value)
        cnt = np.empty(n, np.int32)
        if n:
            ctx.check(ctx.lib.afp_table_fetch_overflow_counts(ctx.h, cnt.ctypes.data))
        # from here on the device table is ahead of the host arrays, whatever happens next
        self._touch()
        self._dev_newer = True
        ctx.table_key = self._dev_key = self._stamp()
        ctx.table_owner = weakref.ref(self)
        self._store_pending = True
        return (ctx, ids, roff, cnt)

    def store_batch_finish(self, token):
        """Second half of store_batch (see store_batch_begin).  Returns the hashes per track."""
        if token is None:
            return []
        ctx, ids, roff, cnt = token
        n = len(cnt)
        if n:
            # overflow entries: random.randint(0, count) is replayed for each, in sequence, on a C
            # copy of CPython's generator; the drawn slots go back and the device applies them (the
            # last entry of a slot wins, as in the reference's sequential loop)
            st = random.getstate()
            state = np.array(st[1], dtype=np.uint32)
            slot = np.empty(n, np.int32)
            ctx.check(ctx.lib.afp_mt_randint_replay(state.ctypes.data, cnt.ctypes.data, n, slot.ctypes.data))
            random.setstate((st[0], tuple(state.tolist()), st[2]))
            ctx.check(ctx.lib.afp_table_apply_slots(ctx.h, slot.ctypes.data, n))
        per_track = np.diff(roff)
        np.add.at(self.__dict__["_hashesperid"], ids, per_track.astype(np.uint32))
        hpi = np.ascontiguousarray(self.hashesperid, dtype=np.uint32)
        ctx.check(ctx.lib.afp_table_set_hashesperid(ctx.h, hpi.ctypes.data if len(hpi) else None, len(hpi)))
        self._store_pending = False
        self._touch()
        ctx.table_key = self._dev_key = self._stamp()      # the device copy IS this version
        return [int(x) for x in per_track]

    def _names_to_ids(self, names):
        """name_to_id(name, add_if_missing=True) (hash_table.py:325-345) for a list of names, without
        the per-name list search: a known name keeps its id, a new one takes the first freed slot,
        else the end of the list."""
        known = {}
        for i, n in enumerate(self.names):
            if n is not None and n not in known:
                known[n] = i
        free = [i for i, n in enumerate(self.names) if n is None]
        free.reverse()
        ids = np.empty(len(names), np.int64)
        hpi = self.__dict__["_hashesperid"]
        grown = []
        for k, name in enumerate(names):
            if not isinstance(name, (str, bytes)):
                ids[k] = name
                continue
            i = known.get(name)
            if i is None:
                if free:
                    i = free.pop()
                    self.names[i] = name
                    hpi[i] = 0
                else:
                    i = len(self.names)
                    self.names.append(name)
                    grown.append(0)
                known[name] = i
            ids[k] = i
        if grown:
            self.hashesperid = np.concatenate([hpi, np.zeros(len(grown), np.uint32)]).astype(np.uint32)
        return ids

    def get_entry(self, hash_):
        """int32 (n,2) [id, time] rows stored under one hash, from the host arrays
        (hash_table.py:140-148; the reference's own version trips over a misspelt attribute)."""
        vals = self.table[hash_, :min(self.depth, int(self.counts[hash_]))].astype(np.int64)
        return np.stack([(vals >> self.maxtimebits) - 1, vals & ((1 << self.maxtimebits) - 1)], axis=1).astype(np.int32)

    def merge(self, ht):
        """Append another table's tracks after ours (hash_table.py:291-323): its ids move up by
        len(self.names); a bucket that still fits keeps every entry (ours first), a bucket that
        does not keeps `depth` entries chosen by np.random.permutation - drawn bucket by bucket in
        ascending hash order, as the reference does, so the same seed gives the same table."""
        if self.maxtimebits != ht.maxtimebits:
            raise AssertionError("tables disagree on maxtimebits (%d vs %d)" % (self.maxtimebits, ht.maxtimebits))
        shift = np.uint32(len(self.names) << self.maxtimebits)
        self.names += ht.names
        self.hashesperid = np.concatenate([self.hashesperid, ht.hashesperid]).astype(np.uint32)
        buckets = np.nonzero(ht.counts)[0]
        have = np.minimum(self.counts[buckets], self.depth).astype(np.int64)       # entries really held
        add = np.minimum(ht.counts[buckets], ht.depth).astype(np.int64)
        fits = have + add <= self.depth
        fb, fh, fa = buckets[fits], have[fits], add[fits]
        for j in range(int(fa.max(initial=0))):                # slot j of the incoming rows, all buckets at once
            m = fa > j
            self.table[fb[m], fh[m] + j] = ht.table[fb[m], j] + shift
        self.counts[fb] = fh + fa
        for b, h, a in zip(buckets[~fits], have[~fits], add[~fits]):
            pool = np.concatenate([self.table[b, :h], ht.table[b, :a] + shift])
            self.table[b] = np.random.permutation(pool)[:self.depth]
            self.counts[b] += ht.counts[b]
        self._touch()

    def name_to_id(self, name, add_if_missing=False):
        """Name -> id (an int is passed through); with add_if_missing a new name takes the first
        freed slot, else the end of the list (hash_table.py:325-345)."""
        if not isinstance(name, (str, bytes)):
            return name
        if name in self.names:
            return self.names.index(name)
        if not add_if_missing:
            raise ValueError("name " + str(name) + " not found")
        if None in self.names:
            slot = self.names.index(None)
            self.names[slot] = name
            self.hashesperid[slot] = 0
            return slot
        self.names.append(name)
        self.hashesperid = np.append(self.hashesperid, [0]).astype(np.uint32)
        return len(self.names) - 1

    def remove(self, name):
        """Drop every entry of `name` (hash_table.py:347-367).  When the device copy is the
        current one (after store_batch) the removal runs there (remove_batch)."""
        if getattr(self, "_dev_newer", False):
            return self.remove_batch([name])
        id_ = self.name_to_id(name)
        mine = (self.table >> np.uint32(self.maxtimebits)) == id_ + 1
        removed = 0
        for hash_ in np.nonzero(np.max(mine, axis=1))[0]:
            n = min(self.depth, int(self.counts[hash_]))
            row = self.table[hash_, :n]
            keep = row[~mine[hash_, :n]]
            self.table[hash_] = 0
            self.table[hash_, :len(keep)] = keep
            self.counts[hash_] = len(keep)
            removed += int(np.sum(mine[hash_]))
        self.names[id_] = None
        self.hashesperid[id_] = 0
        self._touch()
        print("Removed", name, "(", removed, "hashes).")

    def retrieve(self, name):
        """(time, hash) pairs stored for `name` (hash_table.py:369-385), read from the device copy
        when that is the current one (retrieve_batch)."""
        if getattr(self, "_dev_newer", False):
            return self.retrieve_batch([name])[0]
        id_ = self.name_to_id(name)
        tmask = (1 << self.maxtimebits) - 1
        valid = np.arange(self.depth)[None, :] < np.minimum(self.depth, self.counts)[:, None]
        hit = ((self.table >> np.uint32(self.maxtimebits)) == id_ + 1) & valid
        hs, slots = np.nonzero(hit)
        out = np.zeros((len(hs), 2), dtype=np.int32)
        out[:, 0] = self.table[hs, slots] & tmask
        out[:, 1] = hs
        return out

    # ---- batched remove / retrieve on the device table ---------------------------------------
    def remove_batch(self, names):
        """HashTable.remove (hash_table.py:346-364) for a list of tracks (names or ids) in ONE pass
        over the device table.  Leaves table, counts, names and hashesperid as `for n in names:
        self.remove(n)` does and prints the same lines, but checks the whole list first: an unknown
        name, an id outside [0, len(names)) or a track named twice raises ValueError before
        anything changes.  Afterwards the DEVICE copy is the current one (as after store_batch)."""
        self._check_device_edit("remove_batch")
        ids = self._ids_of(names, distinct=True)
        if len(ids) == 0:
            return
        ctx = self._sync_device()
        removed = np.zeros(len(ids), np.int64)
        ctx.check(ctx.lib.afp_table_remove_ids(ctx.h, ids.ctypes.data_as(C.POINTER(C.c_int64)), len(ids),
                                               removed.ctypes.data_as(C.POINTER(C.c_int64))))
        hpi = self.__dict__["_hashesperid"]
        for i in ids:
            self.names[i] = None
            hpi[i] = 0
        self._touch()
        self._dev_newer = True
        ctx.table_key = self._dev_key = self._stamp()      # the device copy IS this version
        ctx.table_owner = weakref.ref(self)
        for name, n in zip(names, removed):
            print("Removed", name, "(", int(n), "hashes).")

    def retrieve_batch(self, names):
        """HashTable.retrieve (hash_table.py:369-385) for a list of tracks (names or ids, repeats
        allowed) in ONE pass over the device table: a list of int32 (n, 2) [time, hash] arrays,
        each equal to retrieve(name).  An unknown name or an id outside [0, len(names)) raises
        ValueError."""
        self._check_device_edit("retrieve_batch")
        ids = self._ids_of(names, distinct=False)
        if len(ids) == 0:
            return []
        ctx = self._sync_device()
        total = C.c_int64(0)
        ctx.check(ctx.lib.afp_table_retrieve_ids(ctx.h, ids.ctypes.data_as(C.POINTER(C.c_int64)), len(ids),
                                                 C.byref(total)))
        rows = np.empty((int(total.value), 2), np.int32)
        off = np.empty(len(ids) + 1, np.int64)
        ctx.check(ctx.lib.afp_fetch_retrieved(ctx.h, rows.ctypes.data if len(rows) else None, 1,
                                              off.ctypes.data_as(C.POINTER(C.c_int64))))
        return [rows[off[k]:off[k + 1]] for k in range(len(ids))]

    def _check_device_edit(self, what):
        # a shard stamp left behind after another table took the device is no shard: _sync_device
        # uploads the whole table again
        if self._shard is not None and _lib.context(self.device).table_key == self._stamp(self._shard):
            raise AfpStateError("the device copy is a shard (restrict_device_ids): cannot %s on it" % what)
        if getattr(self, "_store_pending", False):
            raise AfpStateError("%s: a store_batch_begin was not finished" % what)

    def _ids_of(self, names, distinct):
        """Ids of existing tracks, given by name or by integer id (name_to_id without adding).  A few
        names are searched in the list (names.index: milliseconds each at a million tracks); more
        go through one dict of all names built per call (a few hundred milliseconds at a million)."""
        nids = len(self.names)
        known = None
        if sum(isinstance(n, (str, bytes)) for n in names) > 16:
            try:        # walked backwards, so a name listed twice keeps its first id (names.index)
                known = dict(zip(reversed(self.names), range(nids - 1, -1, -1)))
            except TypeError:                 # a Matlab database marks removed tracks with []
                known = {}
                for i, n in enumerate(self.names):
                    if isinstance(n, (str, bytes)) and n not in known:
                        known[n] = i
        ids = np.empty(len(names), np.int64)
        for k, name in enumerate(names):
            if isinstance(name, (str, bytes)):
                if known is not None:
                    i = known.get(name)
                else:
                    try:
                        i = self.names.index(name)
                    except ValueError:
                        i = None
                if i is None:
                    raise ValueError("name " + str(name) + " not found")
            else:
                i = int(name)
                if not 0 <= i < nids:
                    raise ValueError("track id %d outside [0, %d)" % (i, nids))
            ids[k] = i
        if distinct and len(np.unique(ids)) != len(ids):
            raise ValueError("a track is named twice")
        return ids

    def list(self, print_fn=None):
        """One "<name> (<n> hashes)" line per stored track (hash_table.py:387-391)."""
        emit = print_fn or print
        for track, nhashes in zip(self.names, self.hashesperid):
            if track:
                emit("%s (%s hashes)" % (track, nhashes))

    def totalhashes(self):
        return np.sum(self.counts)

    # ---- persistence (gzip pickle, hash_table.py:178-246) -------------------------------
    def save(self, name, params=None, file_object=None):
        """gzip pickle in the REFERENCE's on-disk format (hash_table.py:178-190): the
        stream names the class `hash_table.HashTable` and carries exactly its attributes,
        so the reference loads files written here and vice versa."""
        if params:
            for key in params:
                self.params[key] = params[key]
        f = file_object if file_object else gzip.open(name, 'wb')
        with _reference_pickle_class() as cls:
            pickle.dump(_as_reference_object(self, cls), f, pickle.HIGHEST_PROTOCOL)
        if not file_object:
            f.close()
        self.dirty = False
        nhashes = int(np.sum(self.counts))
        dropped = nhashes - int(np.sum(np.minimum(self.depth, self.counts)))
        print("Saved fprints for", sum(n is not None for n in self.names),
              "files (", nhashes, "hashes) to", name,
              "(%.2f%% dropped)" % (100.0 * dropped / max(1, nhashes)))

    def load(self, name):
        ext = os.path.splitext(name)[1]
        if ext == '.mat':
            self.load_matlab(name)
        else:
            self.load_pkl(name)
        nhashes = int(np.sum(self.counts))
        dropped = nhashes - int(np.sum(np.minimum(self.depth, self.counts)))
        print("Read fprints for", sum(n is not None for n in self.names),
              "files (", nhashes, "hashes) from", name,
              "(%.2f%% dropped)" % (100.0 * dropped / max(1, nhashes)))

    def load_matlab(self, name):
        """Database written by the Matlab audfprint (hash_table.py:248-285): struct HT_params
        (nhashes, depth, maxtime, hoptime, targetsr, nojenkins, ..., version last), HashTable stored
        depth x buckets, counts, a cell array of names (empty cell = removed track) and the per-track
        hash counts.  Matlab's 1-based ids are what the Python table stores as id + 1, so the entries
        are taken as they are."""
        import scipy.io
        mat = scipy.io.loadmat(name)
        fields = mat['HT_params'][0][0]

        def scalar(k):
            return fields[k][0][0]
        version = scalar(-1)
        if version < 0.9:
            raise AssertionError("Matlab database version %s is older than 0.9" % version)
        if not scalar(5):
            raise AssertionError("Jenkins-hashed Matlab databases are not supported")
        self.hashbits = _bitsfor(scalar(0))
        self.depth = int(scalar(1))
        self.maxtimebits = _bitsfor(scalar(2))
        self.table = np.ascontiguousarray(mat['HashTable'].T, dtype=np.uint32)
        self.counts = np.ascontiguousarray(mat['HashTableCounts'][0], dtype=np.int32)
        self.names = [str(cell[0]) if len(cell) > 0 else [] for cell in mat['HashTableNames'][0]]
        self.hashesperid = np.array(mat['HashTableLengths'][0]).astype(np.uint32)
        self.params = {'mat_version': version, 'hoptime': scalar(3), 'targetsr': scalar(4), 'nojenkins': scalar(5)}
        self.ht_version = HT_VERSION
        self.dirty = False
        self._dev_newer = False
        self._bump()

    def load_pkl(self, name, file_object=None):
        f = file_object if file_object else gzip.open(name, 'rb')
        temp = _RefUnpickler(io.BytesIO(f.read()), encoding='latin1').load()
        if not file_object:
            f.close()
        if temp.ht_version < HT_OLD_COMPAT_VERSION:
            raise ValueError('Version of ' + name + ' is ' + str(temp.ht_version)
                             + ' which is not at least ' + str(HT_OLD_COMPAT_VERSION))
        self.hashbits = temp.hashbits
        self.depth = temp.depth
        self.maxtimebits = temp.maxtimebits if hasattr(temp, 'maxtimebits') else _bitsfor(temp.maxtime)
        table = temp.table
        if temp.ht_version < HT_COMPAT_VERSION:
            print("Loading database version", temp.ht_version, "in compatibility mode.")
            table = table + np.array(1 << self.maxtimebits).astype(np.uint32) * (table != 0)
        self.table = np.ascontiguousarray(table, dtype=np.uint32)
        self.ht_version = HT_VERSION
        self.counts = np.ascontiguousarray(temp.counts, dtype=np.int32)
        self.names = temp.names
        self.hashesperid = np.array(temp.hashesperid).astype(np.uint32)
        self.params = temp.params
        self.dirty = False
        self._dev_newer = False
        self._bump()

    # ---- device copy + probe --------------------------------------------------------
    def _stamp(self, shard=None):
        return (self._token, self._version, int(self.hashbits), int(self.depth), int(self.maxtimebits), shard)

    def _sync_device(self):
        """Upload table/counts/hashesperid if they changed since the last upload."""
        ctx = _lib.context(self.device)
        if self._shard is not None and ctx.table_key == self._stamp(self._shard):
            return ctx              # device copy is this table's shard
        if ctx.table_key != self._stamp():
            self._shard = None
            # the device may hold ANOTHER table's only copy of its device-side inserts: save it first
            owner = ctx.table_owner() if getattr(ctx, "table_owner", None) else None
            if owner is not None and owner is not self and getattr(owner, "_dev_newer", False):
                owner._pull_device()
            ctx.table_owner = None
            table = np.ascontiguousarray(self.table, dtype=np.uint32)     # (pulls the device copy first if it is newer)
            counts = np.ascontiguousarray(self.counts, dtype=np.int32)
            hpi = np.ascontiguousarray(self.hashesperid, dtype=np.uint32)
            if table.shape != (1 << int(self.hashbits), int(self.depth)) or counts.shape != (1 << int(self.hashbits),):
                raise ValueError("table/counts shapes do not match hashbits/depth")
            ctx.check(ctx.lib.afp_table_upload(ctx.h, table.ctypes.data, counts.ctypes.data, int(self.hashbits),
                                               int(self.depth), int(self.maxtimebits),
                                               hpi.ctypes.data if len(hpi) else None, len(hpi), 1))
            ctx.table_key = self._stamp()
        return ctx

    def restrict_device_ids(self, id_lo, id_hi):
        """Keep only entries of ids in [id_lo, id_hi) in the DEVICE copy (a table shard,
        SURVEY.md §8e); the host arrays are untouched.  Any later mutation (or another
        restrict) starts again from the full table."""
        ctx = _lib.context(self.device)
        ctx.table_key = None                      # force a fresh upload of the whole table
        self._shard = None
        ctx = self._sync_device()
        ctx.check(ctx.lib.afp_table_restrict_ids(ctx.h, int(id_lo), int(id_hi)))
        self._shard = (int(id_lo), int(id_hi))
        ctx.table_key = self._stamp(self._shard)
        return ctx

    def _pull_device(self):
        """Refresh the host arrays from the device copy after device-side inserts."""
        ctx = _lib.context(self.device)
        if ctx.table_key != getattr(self, "_dev_key", None):
            raise AfpStateError("the device table that holds this table's inserts was replaced by another upload")
        table = np.empty((1 << int(self.hashbits), int(self.depth)), np.uint32)
        counts = np.empty(1 << int(self.hashbits), np.int32)
        ctx.check(ctx.lib.afp_table_download(ctx.h, table.ctypes.data, counts.ctypes.data))
        self.__dict__["_table"], self.__dict__["_counts"] = table, counts
        self._dev_newer = False

    def get_hits(self, hashes):
        """[time, hash] rows -> int32 (nhits,4) [id, dtime, hash, time] rows in
        (query row, slot) order (hash_table.py:150-176)."""
        q = np.ascontiguousarray(np.asarray(hashes, dtype=np.int32).reshape(-1, 2))
        ctx = self._sync_device()
        n = C.c_int64(0)
        ctx.check(ctx.lib.afp_get_hits(ctx.h, q.ctypes.data if len(q) else None, len(q), 1, C.byref(n)))
        hits = np.empty((int(n.value), 4), np.int32)
        ctx.check(ctx.lib.afp_fetch_hits(ctx.h, hits.ctypes.data if len(hits) else None, 1))
        return hits
