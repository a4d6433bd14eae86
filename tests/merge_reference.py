"""HashTable.merge (reference hash_table.py:291-323) as a plain per-bucket loop, the statement the
device merge (csrc/afp_table_merge.cu) is held to by tests/test_gpu_table_merge.py;
tests/test_table_merge_cpu.py pins it to the table the reference merged and to the host mirror.

A state is any object with `hashbits`, `depth`, `maxtimebits`, `table`, `counts`, `names` and
`hashesperid`, as in tests/table_reference.py (a State or an audfprint_b200.HashTable)."""
import numpy as np


def merge(state, other, rng=np.random):
    """Append `other`'s tracks after ours: its ids move up by len(names) (uint32 arithmetic on the
    entries).  Bucket by bucket, in ascending order over the non-zero counts of `other`: the pool is
    our first min(count, depth) entries followed by its first min(count, its depth) shifted ones; a
    pool that fits is written from slot 0 (later slots keep their values) and its length becomes the
    count; a larger one is rng.permutation(pool)[:depth] and the count grows by other's raw count."""
    assert state.maxtimebits == other.maxtimebits
    ncurrent = len(state.names)
    state.names += list(other.names)
    state.hashesperid = np.append(state.hashesperid, other.hashesperid).astype(np.uint32)
    idoffset = ncurrent << state.maxtimebits
    for b in np.nonzero(other.counts)[0]:
        mine = [int(v) for v in state.table[b, :min(int(state.counts[b]), state.depth)]]
        theirs = [(int(v) + idoffset) & 0xffffffff for v in other.table[b, :min(int(other.counts[b]), other.depth)]]
        pool = np.array(mine + theirs, np.uint32)
        if len(pool) <= state.depth:
            state.table[b, :len(pool)] = pool
            state.counts[b] = len(pool)
        else:
            state.table[b] = rng.permutation(pool)[:state.depth]
            state.counts[b] = int(state.counts[b]) + int(other.counts[b])
