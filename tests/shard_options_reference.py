"""Host statement of what ONE shard of an id-range sharded table publishes when the matcher's
exact_count / find_time_range options are on (afp_match_options_shard_rank / _finish +
afp_shard_pack), built from the oracle's pieces.

It differs from the whole-table finish (oracle.match_hashes) in the three places that are not
local to a shard:
  * every candidate the shard publishes (rank < min(#ids, search_depth)) is finished, not only
    the ranks below the shard's own n_above - the merge drops global ranks >= D;
  * the (qtime, hash) keys are packed with `timebits`, the caller's key width: the one of the
    query's largest qtime over the WHOLE table (the oracle's pair_bits reads it from the hits it is
    given, which on a shard are the shard's alone);
  * a quantile index outside its support is recorded (the smallest failing local rank), not raised.
"""
import numpy as np

from oracle import afp_oracle as orc


def key_bits(qmax: int) -> int:
    """The reference's key width for a query whose largest qtime is qmax (pair_bits' expression)."""
    return max(1, int(np.ceil(np.log(max(1, int(qmax))) / np.log(2))))


def query_qmax(hits: np.ndarray) -> int:
    """Largest qtime of a query's hits, 0 without hits (the device's starting value)."""
    return int(hits[:, 3].max()) if len(hits) else 0


def _time_range(hits, id_, mode, window, quant):
    """orc.time_range, or None where the reference raises IndexError."""
    try:
        return orc.time_range(hits, id_, mode, window, quant)
    except IndexError:
        return None


def shard_options_record(hits, hpi, lo, hi, window, thresh, sdepth, exact, trange, quant, timebits,
                         max_alignments_per_id=100):
    """One query on shard [lo, hi).  hits: the query's hits over the WHOLE table (get_hits).
    Returns {"n_above", "cand" (k,3) [id, raw, weight], "rows" (r,7) with LOCAL ranks,
    "fail" (smallest local rank whose quantile read failed, -1 = none)}."""
    hits = hits[(hits[:, 0] >= lo) & (hits[:, 0] < hi)]
    empty = {"n_above": 0, "cand": np.zeros((0, 3)), "rows": np.zeros((0, 7), np.int32), "fail": -1}
    if len(hits) == 0 or sdepth <= 0:
        if len(hits):
            ids, raw = np.unique(hits[:, 0], return_counts=True)
            empty["n_above"] = int(np.count_nonzero(raw > thresh))
        return empty
    ids, raw = np.unique(hits[:, 0], return_counts=True)
    wtd = raw / hpi[ids].astype(float)
    order = np.lexsort((-ids, -wtd))[:sdepth]
    cids, craw = ids[order], raw[order]
    fail = []
    if exact:
        rows = []
        for rank, (id_, r) in enumerate(zip(cids, craw)):
            dts = hits[hits[:, 0] == id_, 1].astype(np.int64)
            base = int(dts.min())
            hist = np.bincount(dts - base)
            for k in np.nonzero(orc.local_max_mask(hist) & (hist >= thresh))[0]:
                mode = int(k) + base
                sup = orc.support_rows(hits, int(id_), mode, window)
                n = len(set(int(t) + (int(h) << timebits) for t, h in zip(sup[:, 3], sup[:, 2])))
                if n < thresh:
                    continue
                lo_t = hi_t = 0
                if trange:
                    tr = _time_range(hits, int(id_), mode, window, quant)
                    if tr is None:
                        fail.append(rank)
                    else:
                        lo_t, hi_t = tr
                rows.append([int(id_), n, mode, int(r), rank, lo_t, hi_t])
        rows = np.array(rows, np.int32).reshape(-1, 7)
    else:
        rows = orc.offset_histogram_rows(hits, cids, craw, window, thresh, max_alignments_per_id)
        if trange:
            for row in rows:
                tr = _time_range(hits, int(row[0]), int(row[2]), window, quant)
                if tr is None:
                    fail.append(int(row[4]))
                    row[5] = row[6] = 0
                else:
                    row[5], row[6] = tr
    return {"n_above": int(np.count_nonzero(raw > thresh)),
            "cand": np.stack([cids, craw, wtd[order]], axis=1).astype(np.float64),
            "rows": rows, "fail": min(fail) if fail else -1}


def batch_arrays(recs, sdepth):
    """Per-query records -> the arrays pack_shard_batch takes (cand, counts, rows, row_off, fail)."""
    nq, sd = len(recs), max(int(sdepth), 1)
    cand = np.zeros((nq, sd, 3))
    cnts = np.zeros((nq, 2), np.int32)
    roff = np.zeros(nq + 1, np.int64)
    for i, r in enumerate(recs):
        k = len(r["cand"])
        cand[i, :k] = r["cand"]
        cnts[i] = (k, r["n_above"])
        roff[i + 1] = roff[i] + len(r["rows"])
    rows = np.concatenate([r["rows"] for r in recs]) if recs else np.zeros((0, 7), np.int32)
    return cand, cnts, rows.astype(np.int32), roff, np.array([r["fail"] for r in recs], np.int64)


def pack_shard(recs, sdepth, row_cap):
    """The records afp_shard_pack writes after an options finish on this shard."""
    from audfprint_b200 import dist as afd
    cand, cnts, rows, roff, fail = batch_arrays(recs, sdepth)
    return afd.pack_shard_batch(cand, cnts, rows, roff, row_cap, fail_rank=fail)
