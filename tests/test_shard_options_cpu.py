"""CPU: exact_count / find_time_range on a table sharded by track-id range, stated on the host.
Each shard's records come from the host statement (tests/shard_options_reference.py) with the
WHOLE table's key width; the per-query maxima are all-reduced and the records all-gathered over
gloo at world size 2, then merged (dist.merge_shard_batch).  The merged rows must be the oracle's
single-table rows."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from audfprint_b200 import dist as afd
from oracle import afp_oracle as orc
from tests import cases
from tests import shard_options_reference as sor
from tests.conftest import expand_table, GOLDEN

MODES = ((True, False), (False, True), (True, True))
RCAP = 2048            # the host merge has no shared-memory bound on nshards * row_cap


def _merged_vs_oracle(table, counts, hashbits, depth, mtb, hpi, qs, hits, shards_mine, nshards, window, thresh,
                      sdepth, exact, trange, quant):
    """This rank's shards (shards_mine) through the host statement; qmax all-reduced and records
    all-gathered when a process group is up.  Returns True when every query equals the oracle."""
    nids = len(hpi)
    qmax = torch.tensor([sor.query_qmax(h[(h[:, 0] >= afd.id_range(nids, s, nshards)[0]) &
                                          (h[:, 0] < afd.id_range(nids, s, nshards)[1])])
                         for h in hits for s in shards_mine] or [0], dtype=torch.int64)
    qmax = qmax.reshape(len(hits), -1).max(dim=1).values if len(shards_mine) else torch.zeros(len(hits), dtype=torch.int64)
    if afd.world()[1] > 1:
        dist.all_reduce(qmax, op=dist.ReduceOp.MAX)
    bits = [sor.key_bits(int(v)) for v in qmax]
    mine = {}
    for s in shards_mine:
        lo, hi = afd.id_range(nids, s, nshards)
        recs = [sor.shard_options_record(h, hpi, lo, hi, window, thresh, sdepth, exact, trange, quant, b)
                for h, b in zip(hits, bits)]
        mine[s] = sor.pack_shard(recs, sdepth, RCAP)
    everyone = {}
    for part in afd.gather_objects(mine):
        everyone.update(part)
    gathered = np.stack([everyone[s] for s in range(nshards)])
    rows, off = afd.merge_shard_batch(gathered, sdepth, RCAP)
    ok = True
    for qi, q in enumerate(qs):
        got = rows[off[qi]:off[qi + 1]]
        got = got[np.argsort(-got[:, 1], kind="stable")]
        want = orc.match_hashes(table, counts, hashbits, depth, mtb, hpi, q, window=window, threshcount=thresh,
                                search_depth=sdepth, exact_count=exact, find_time_range=trange, quantile=quant)
        ok = ok and np.array_equal(got, want)
    return ok


def _golden_queries(gm, db):
    table, counts, hashbits, depth, mtb, hpi = expand_table(gm, db)
    qs = [gm["q%d_%s/q" % (j, tag)] for j in range(cases.DB_QUERIES) for tag in ("clean", "noisy")]
    hits = [orc.get_hits(table, counts, hashbits, depth, mtb, q) for q in qs]
    return (table, counts, hashbits, depth, mtb, hpi), qs, hits


CONFIGS = ((1, 5, 100, 0.02), (2, 1, 4, 0.05), (0, 2, 100, 0.5), (2, 2, 10, 0.0))


def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        gm = np.load(os.path.join(GOLDEN, "match.npz"))
        ok = True
        for db in ("db", "db2"):
            tab, qs, hits = _golden_queries(gm, db)
            for nshards in (2, 3, 5):
                shards_mine = [s for s in range(nshards) if s % world == rank]
                for k, (exact, trange) in enumerate(MODES):
                    window, thresh, sdepth, quant = CONFIGS[(k + nshards) % len(CONFIGS)]
                    ok = ok and _merged_vs_oracle(*tab, qs, hits, shards_mine, nshards, window, thresh, sdepth,
                                                  exact, trange, quant)
        out.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_sharded_options_world2_gloo():
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, out)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(600)
            assert p.exitcode == 0
        res = sorted(out.get(timeout=10) for _ in procs)
        assert res == [(0, True), (1, True)]
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()


@pytest.mark.parametrize("db", ["db", "db2"])
def test_every_config_single_process(golden_match, db):
    """All shards in one process (no process group), at 2, 3 and 5 shards: every option mode with
    the configurations the world-2 run does not give it."""
    tab, qs, hits = _golden_queries(golden_match, db)
    for nshards in (2, 3, 5):
        for k, (exact, trange) in enumerate(MODES):
            for window, thresh, sdepth, quant in (CONFIGS[(k + nshards + 1) % 4], CONFIGS[(k + nshards + 2) % 4]):
                assert _merged_vs_oracle(*tab, qs, hits, list(range(nshards)), nshards, window, thresh, sdepth,
                                         exact, trange, quant), (nshards, exact, trange, window, thresh, sdepth)


# ---- the key width is the whole table's ------------------------------------------------------
HB, CDEPTH, MTB = 12, 64, 13


def _np_table(tracks):
    nb = 1 << HB
    table = np.zeros((nb, CDEPTH), np.uint32)
    counts = np.zeros(nb, np.int32)
    hpi = np.zeros(len(tracks), np.uint32)
    for i, th in enumerate(tracks):
        for t, h in np.asarray(th, np.int64).reshape(-1, 2):
            b = h & (nb - 1)
            table[b, counts[b]] = ((i + 1) << MTB) | (t & ((1 << MTB) - 1))
            counts[b] += 1
        hpi[i] = len(th)
    return table, counts, HB, CDEPTH, MTB, hpi


def power_of_two_case():
    """Track 0's largest query time is 2^11: at 11 key bits (2^11, h) and (0, h + 1) collide.  Track
    1 holds the query's real largest time (5000): at the whole table's 13 bits they do not."""
    h = 900
    col = [(1 << 11, h, 5), (0, h + 1, 5), (100, h + 2, 5)]
    other = [(5000, 950, 1), (5001, 951, 1)]
    tracks = [[(t + d, hh) for t, hh, d in col], [(t + d, hh) for t, hh, d in other]]
    q = np.array([(t, hh) for t, hh, _ in col + other], np.int32)
    return _np_table(tracks), q


def test_shard_local_key_width_differs():
    (table, counts, hashbits, depth, mtb, hpi), q = power_of_two_case()
    hits = orc.get_hits(table, counts, hashbits, depth, mtb, q)
    assert sor.key_bits(sor.query_qmax(hits)) == 13 and sor.key_bits(1 << 11) == 11
    want = orc.match_hashes(table, counts, hashbits, depth, mtb, hpi, q, window=0, threshcount=1,
                            search_depth=100, exact_count=True)
    assert want[want[:, 0] == 0][0, 1] == 3
    nshards = 2
    assert [afd.id_range(2, s, nshards) for s in range(2)] == [(0, 1), (1, 2)]      # one track per shard
    for local in (False, True):
        recs = []
        for s in range(nshards):
            lo, hi = afd.id_range(2, s, nshards)
            hs = hits[(hits[:, 0] >= lo) & (hits[:, 0] < hi)]
            bits = sor.key_bits(sor.query_qmax(hs if local else hits))
            recs.append(sor.pack_shard([sor.shard_options_record(hits, hpi, lo, hi, 0, 1, 100, True, False, 0.0,
                                                                 bits)], 100, RCAP))
        rows, off = afd.merge_shard_batch(np.stack(recs), 100, RCAP)
        count0 = rows[rows[:, 0] == 0][0, 1]
        assert count0 == (2 if local else 3)
        if not local:
            assert np.array_equal(rows[np.argsort(-rows[:, 1], kind="stable")], want)


def test_status_word_decisions():
    """check_shard_status: a failed quantile read raises only inside the global top-D; an overflow
    raises ValueError naming the row count the shard produced."""
    sd = 4

    def rec(n_above, ids, wts, nrows=0, status=0):
        r = np.zeros(1, afd.record_dtype(sd, 2))
        r["hdr"][0] = (n_above, len(ids), nrows, status)
        r["id"][0, :len(ids)], r["w"][0, :len(ids)], r["raw"][0, :len(ids)] = ids, wts, 1
        return r
    a = rec(1, [5, 3], [0.9, 0.1])
    b_fail1 = rec(0, [7, 6], [0.5, 0.2], status=(1 + 1) << 1)       # local rank 1: weight 0.2 -> global rank 2
    afd.check_shard_status(np.stack([a, b_fail1]), 100)             # D = 1: not reached
    with pytest.raises(IndexError):
        afd.check_shard_status(np.stack([a, rec(2, [7, 6], [0.5, 0.2], status=(1 + 1) << 1)]), 100)   # D = 3
    with pytest.raises(IndexError):
        afd.check_shard_status(np.stack([a, rec(0, [7, 6], [0.95, 0.2], status=(0 + 1) << 1)]), 100)  # global rank 0
    with pytest.raises(ValueError, match="produced 9 rows"):
        afd.check_shard_status(np.stack([a, rec(0, [7, 6], [0.5, 0.2], nrows=9, status=afd.STATUS_OVERFLOW)]), 100)
