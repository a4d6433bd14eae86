"""The multi-process ingest's statement (tests/ingest_merge_reference.py) and the host mirror
against what the reference's own multiproc_add built (tests/golden/ingest_merge.npz): table,
counts, names, hashesperid, report lines and the parent's next np.random draw, for ncores 1, 2, 3
and 5, `new` into an empty table and `add` into a base with a removed track."""
import os
import random

import numpy as np
import pytest

from audfprint_b200 import HashTable
from tests import ingest_merge_reference as im
from tests import table_reference as ref
from tests.conftest import GOLDEN


@pytest.fixture(scope="module")
def golden_ingest():
    return np.load(os.path.join(GOLDEN, "ingest_merge.npz"))


def _check(st, want, key, lines=None, nxt=None):
    assert np.array_equal(st.table, want[key + "/table"]), key
    assert np.array_equal(st.counts, want[key + "/counts"]), key
    assert list(st.names) == im.golden_names(want, key), key
    assert np.array_equal(st.hashesperid, want[key + "/hashesperid"]), key
    assert np.asarray(st.hashesperid).dtype == np.uint32
    if lines is not None:
        assert lines == want[key + "/report"].tolist(), key
    if nxt is not None:
        assert nxt == float(want[key + "/np_next"]), key


@pytest.mark.parametrize("mode,ncores", im.CASES)
def test_statement_equals_the_reference(golden_match, golden_ingest, mode, ncores):
    want = golden_ingest
    files = im.fixture_files(golden_match, mode)
    base = im.golden_base(want, mode)
    np.random.seed(im.NP_SEED)
    lines = im.multiproc_add(base, files, ncores, [im.SEED + r for r in range(ncores)])
    _check(base, want, "%s_%d" % (mode, ncores), lines, np.random.random())


@pytest.mark.parametrize("mode,ncores", im.CASES)
def test_host_mirror_equals_the_reference(golden_match, golden_ingest, mode, ncores):
    """HashTable.store per worker from its own seed, then HashTable.merge in worker order."""
    want = golden_ingest
    files = im.fixture_files(golden_match, mode)
    ht = ref.mirror(im.golden_base(want, mode))
    workers = []
    for r, idx in enumerate(im.deal(len(files), ncores)):
        random.seed(im.SEED + r)
        w = HashTable(hashbits=im.HASHBITS, depth=im.DEPTH, maxtime=1 << im.MAXTIMEBITS)
        for i in idx:
            w.store(*files[i])
        workers.append(w)
    np.random.seed(im.NP_SEED)
    lines = []
    for r, w in enumerate(workers):
        lines.append("hash_table %d has %d files %d hashes" % (r, len(w.names), int(w.counts.sum())))
        ht.merge(w)
    _check(ht, want, "%s_%d" % (mode, ncores), lines, np.random.random())


def test_the_fixture_reaches_every_trap(golden_match, golden_ingest):
    """Workers whose buckets overflow, merges that overflow, a base with a freed slot, a file with no
    hashes and workers with no files - and a per-worker table whose raw counts exceed depth, which
    the merge into an empty table clips (the parent cannot adopt worker 0's table as its own)."""
    want = golden_ingest
    files = im.fixture_files(golden_match)
    ws = [im.worker_table([files[i] for i in idx], im.HASHBITS, im.DEPTH, im.MAXTIMEBITS,
                          random.Random(im.SEED + r)) for r, idx in enumerate(im.deal(len(files), 5))]
    assert all((w.counts > im.DEPTH).any() for w in ws)
    assert (want["new_1/counts"] <= im.DEPTH).all() and (want["new_2/counts"] > im.DEPTH).any()
    one = im.worker_table(files, im.HASHBITS, im.DEPTH, im.MAXTIMEBITS, random.Random(im.SEED))
    assert not np.array_equal(one.counts, want["new_1/counts"])
    assert None in im.golden_names(want, "base")
    assert "silence" in im.golden_names(want, "new_5")
    assert want["few_5/report"].tolist()[3:] == ["hash_table 3 has 0 files 0 hashes",
                                                 "hash_table 4 has 0 files 0 hashes"]
