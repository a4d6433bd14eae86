"""Golden vectors for the multi-process ingest, produced by the LIVE reference's own
`audfprint.multiproc_add` (audfprint.py:199-235): worker processes build one table each from their
share of the files (make_ht_from_list) and the parent merges them in worker order
(hash_table.py:291-323).

Two things are pinned so that the run is reproducible:
  * each forked worker would reseed `random` from OS entropy; make_ht_from_list is wrapped so that
    worker r seeds it with SEED + r (r = the index of its first file modulo ncores; a worker
    without files draws nothing);
  * the analyzer is a stub whose wavfile2hashes returns stored track hashes (tests/golden/match.npz),
    so only the table building is under test.
The cases (tests/ingest_merge_reference.py): 2^10 x 6, ncores 1, 2, 3 and 5, `new` into an empty
table and `add` into a base that the reference built and removed a track from, plus 3 files on 5
workers.

Needs a checkout of the reference (dpwe/audfprint) named by $AFP_REFERENCE:
    AFP_REFERENCE=<checkout> python oracle/make_golden_ingest_merge.py
Only OUTPUT ARRAYS of the reference are stored; no reference source is copied.
"""
from __future__ import annotations

import os
import random
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ["AFP_REFERENCE"])
sys.modules.setdefault("docopt", types.ModuleType("docopt"))    # the CLI parser; not used here

import audfprint as ref_cli             # noqa: E402  (the reference)
import hash_table as ref_ht             # noqa: E402

from tests import ingest_merge_reference as im     # noqa: E402  (constants and file list only)

OUT = os.path.join(ROOT, "tests", "golden")


class StubAnalyzer(object):
    def __init__(self, files):
        self.rows = dict(files)

    def wavfile2hashes(self, filename):
        return self.rows[filename]


def seeded_workers(order, ncores):
    make = ref_cli.make_ht_from_list

    def make_seeded(analyzer, filelist, hashbits, depth, maxtime, pipe=None):
        if filelist:
            random.seed(im.SEED + order[filelist[0]] % ncores)
        return make(analyzer, filelist, hashbits, depth, maxtime, pipe)
    return make_seeded


def record(out, key, ht):
    out[key + "/table"] = np.asarray(ht.table, np.uint32).copy()
    out[key + "/counts"] = np.asarray(ht.counts, np.int32).copy()
    out[key + "/hashesperid"] = np.asarray(ht.hashesperid, np.uint32).copy()
    out[key + "/names"] = np.array(["" if n is None else n for n in ht.names])


def main():
    gm = np.load(os.path.join(OUT, "match.npz"))
    out = {}
    random.seed(im.BASE_SEED)
    base = ref_ht.HashTable(hashbits=im.HASHBITS, depth=im.DEPTH, maxtime=1 << im.MAXTIMEBITS)
    for i in im.BASE_TRACKS:
        base.store("track%d" % i, gm["track%d/hashes" % i])
    base.remove(im.BASE_REMOVED)
    record(out, "base", base)
    orig = ref_cli.make_ht_from_list
    for mode, ncores in im.CASES:
        files = im.fixture_files(gm, mode)
        order = {name: i for i, (name, _) in enumerate(files)}
        ht = ref_ht.HashTable(hashbits=im.HASHBITS, depth=im.DEPTH, maxtime=1 << im.MAXTIMEBITS)
        if mode == "add":
            ht.table, ht.counts = base.table.copy(), base.counts.copy()
            ht.names, ht.hashesperid = list(base.names), base.hashesperid.copy()
        lines = []
        ref_cli.make_ht_from_list = seeded_workers(order, ncores)
        try:
            np.random.seed(im.NP_SEED)
            ref_cli.multiproc_add(StubAnalyzer(files), ht, [n for n, _ in files], lines.extend, ncores)
            nxt = np.random.random()
        finally:
            ref_cli.make_ht_from_list = orig
        key = "%s_%d" % (mode, ncores)
        record(out, key, ht)
        out[key + "/report"] = np.array(lines)
        out[key + "/np_next"] = np.float64(nxt)
        print(key, "entries", int(ht.counts.sum()), "overfull buckets", int(np.sum(ht.counts > im.DEPTH)),
              "names", len(ht.names), lines)
    np.savez_compressed(os.path.join(OUT, "ingest_merge.npz"), **out)


if __name__ == "__main__":
    main()
