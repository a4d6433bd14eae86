"""Multi-GPU plumbing: one process per GPU, `torch.distributed` for the rendezvous.

The reference's only parallelism is sharding the FILE LIST over OS processes
(`multiproc_add`, audfprint.py:199-235: file ix goes to process ix % ncores) and
pickling results back.  The same shape is used here:

* fingerprinting: file i -> rank i % world; NO data-path collective (results are
  per-file and gathered as host objects only if the caller asks for them);
* matching, table replicated (419 MB << 80 GB): query j -> rank j % world; no
  collective;
* matching, table sharded by track-id range (SURVEY.md §8e, BASELINE configs[4]):
  every rank sees every query, computes the candidate list and result rows of
  ITS ids, and ONE all-gather of fixed-size per-query records merges them:
  `merge_sharded_results` below is exact because an id inside the global top-D
  (D = min(sum n_above, search_depth)) is inside its own shard's local top-D.

Nothing here computes on the CPU; it only moves and merges small result records.
"""
from __future__ import annotations

import numpy as np


def world():
    """(rank, world_size) of the default process group, (0, 1) when not initialised."""
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return dist.get_rank(), dist.get_world_size()
    except ImportError:
        pass
    return 0, 1


def shard_indices(n: int, rank: int, world_size: int) -> np.ndarray:
    """Indices of the items rank `rank` owns: i % world == rank (audfprint.py:211-214)."""
    return np.arange(rank, n, world_size, dtype=np.int64)


def id_range(nids: int, rank: int, world_size: int):
    """Contiguous track-id range [lo, hi) of a rank's table shard."""
    lo = (nids * rank) // world_size
    hi = (nids * (rank + 1)) // world_size
    return lo, hi


def gather_objects(obj, group=None):
    """all_gather of small host objects (result lists); identity without a process group."""
    rank, ws = world()
    if ws == 1:
        return [obj]
    import torch.distributed as dist
    out = [None] * ws
    dist.all_gather_object(out, obj, group=group)
    return out


def interleave_shards(per_rank_lists, n: int):
    """Inverse of shard_indices: per_rank_lists[r][k] is the result of item r + k*world."""
    ws = len(per_rank_lists)
    out = [None] * n
    for r, lst in enumerate(per_rank_lists):
        for k, v in enumerate(lst):
            out[r + k * ws] = v
    return out


# ---- sharded-table match: merge of per-shard records ---------------------------------
def merge_sharded_results(shard_records, search_depth: int):
    """Merge one query's per-shard records into the rows a single table would give.

    shard_records: list over shards of dicts with
        n_above  int                      #ids of the shard with raw > threshcount
        cand     float64/int64 (k,3)      the shard's local top-k ids by (weight desc, id desc):
                                          columns [id, raw, weight]; k = min(#distinct ids, search_depth)
        rows     int32 (r,7)              rows of those candidates, column 4 = LOCAL rank
    Returns int32 (R,7) rows with column 4 = global rank, in global rank order (the order
    Matcher._approx_match_counts emits them, audfprint_match.py:279-311), before the final
    sort by count (:335).

    Exactness: the global candidate list is the top-D of all distinct ids by weight,
    D = min(sum n_above, search_depth) (audfprint_match.py:139-146).  Any id in it has fewer
    than D ids above it globally, hence fewer than D above it in its own shard, so it is in
    that shard's published list; and every id outranking it is in the global top-D too, so the
    position in the merged lists IS its global rank."""
    depth = min(int(sum(r["n_above"] for r in shard_records)), int(search_depth))
    if depth <= 0:
        return np.zeros((0, 7), np.int32)
    ids, wts, src = [], [], []
    for s, rec in enumerate(shard_records):
        c = np.asarray(rec["cand"], dtype=np.float64).reshape(-1, 3)
        ids.append(c[:, 0].astype(np.int64))
        wts.append(c[:, 2])
        src.append(np.full(len(c), s))
    ids, wts = np.concatenate(ids), np.concatenate(wts)
    order = np.lexsort((-ids, -wts))[:depth]            # weight desc, then id desc
    grank = {int(ids[o]): g for g, o in enumerate(order)}
    rows = []
    for rec in shard_records:
        for row in np.asarray(rec["rows"], dtype=np.int32).reshape(-1, 7):
            g = grank.get(int(row[0]))
            if g is not None:
                r2 = row.copy()
                r2[4] = g
                rows.append(r2)
    if not rows:
        return np.zeros((0, 7), np.int32)
    rows = np.stack(rows)
    # rank-major; rows of one id keep the order the kernel emitted them in
    return rows[np.argsort(rows[:, 4], kind="stable")]


# ---- the one exchange step of the sharded-table match --------------------------------
# Wire format = the byte records of csrc/afp_shard.cu (afp_shard_pack / afp_shard_merge): per
# query  int32 {n_above, ncand, nrows, 0}; f64 weight[sd]; uint32 id[sd]; uint32 raw[sd];
# int32 rows[row_cap][7].  The NumPy pack / merge below are the host-side statement of the same
# format and the same merge: they serve the CPU (gloo) tests and check the device kernels; the
# product path (match_sharded_batch) packs, gathers and merges on the device.
def record_dtype(search_depth: int, row_cap: int) -> np.dtype:
    sd = max(int(search_depth), 1)
    if row_cap < 2 or row_cap % 2:
        raise ValueError("row_cap must be even and >= 2")
    return np.dtype([("hdr", "<i4", (4,)), ("w", "<f8", (sd,)), ("id", "<u4", (sd,)), ("raw", "<u4", (sd,)),
                     ("rows", "<i4", (row_cap, 7))])


def pack_shard_records(records, search_depth: int, row_cap: int) -> np.ndarray:
    """List of per-query dicts (match_batch_shard) -> structured array (nq,) in the wire format."""
    out = np.zeros(len(records), record_dtype(search_depth, row_cap))
    sd = out.dtype["w"].shape[0]
    for i, r in enumerate(records):
        c = np.asarray(r["cand"], np.float64).reshape(-1, 3)[:sd]
        rows = np.asarray(r["rows"], np.int32).reshape(-1, 7)
        if len(rows) > row_cap:
            raise ValueError("a shard produced %d rows for one query, row_cap is %d" % (len(rows), row_cap))
        out["hdr"][i, :3] = (r["n_above"], len(c), len(rows))
        out["id"][i, :len(c)], out["raw"][i, :len(c)], out["w"][i, :len(c)] = c[:, 0], c[:, 1], c[:, 2]
        out["rows"][i, :len(rows)] = rows
    return out


def unpack_shard_records(buf: np.ndarray, search_depth: int = None, row_cap: int = None):
    recs = []
    for r in buf:
        nc, nr = int(r["hdr"][1]), int(r["hdr"][2])
        cand = np.stack([r["id"][:nc].astype(np.float64), r["raw"][:nc].astype(np.float64), r["w"][:nc]], axis=1)
        recs.append({"n_above": int(r["hdr"][0]), "cand": cand, "rows": r["rows"][:nr].copy()})
    return recs


def _allgather_bytes(mine: np.ndarray, group=None) -> np.ndarray:
    """all_gather of one structured array per rank -> (world, nq) structured array."""
    rank, ws = world()
    if ws == 1:
        return mine[None]
    import torch
    import torch.distributed as dist
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")
    t = torch.from_numpy(np.ascontiguousarray(mine).view(np.uint8).reshape(len(mine), -1)).to(dev)
    out = torch.empty((ws * t.shape[0], t.shape[1]), dtype=torch.uint8, device=dev)
    dist.all_gather_into_tensor(out, t, group=group)
    return out.cpu().numpy().view(mine.dtype).reshape(ws, len(mine))


def allgather_shard_records(records, search_depth: int, row_cap: int = 16, group=None):
    """ONE all-gather (NCCL over NVLink when the group is nccl, gloo on CPU) of the packed
    per-query records of every shard.  Returns per_shard[s][q] record dicts."""
    gathered = _allgather_bytes(pack_shard_records(records, search_depth, row_cap), group)
    return [unpack_shard_records(g) for g in gathered]


def match_sharded(matcher, ht, queries, row_cap: int = 16, group=None):
    """Sharded-table match of `queries` (every rank passes the same list): this rank's
    device table must already be restricted to its id range
    (HashTable.restrict_device_ids(*id_range(nids, rank, world))).  Returns the rows a
    single table gives, on every rank.  Per-query host objects (API convenience; the batch form
    below is the throughput path)."""
    mine = matcher.match_batch_shard(ht, queries)
    shards = allgather_shard_records(mine, matcher.search_depth, row_cap, group)
    out = []
    for qi in range(len(queries)):
        rows = merge_sharded_results([s[qi] for s in shards], matcher.search_depth)
        out.append(rows[(-rows[:, 1]).argsort(), ])          # audfprint_match.py:335
    return out


# ---- vectorised host statement of pack / merge (tests; checks the device kernels) --------
def pack_shard_batch(cand, counts, rows, row_off, row_cap: int) -> np.ndarray:
    """The wire records built without a Python loop from what afp_fetch_match_candidates /
    afp_fetch_match_rows return: cand (nq, sd, 3) f64, counts (nq, 2) i32 [entries, n_above],
    rows (R, 7) i32, row_off (nq+1)."""
    nq, sd = cand.shape[0], cand.shape[1]
    nrows = np.diff(row_off)
    if nq and nrows.max(initial=0) > row_cap:
        raise ValueError("a shard produced %d rows for one query, row_cap is %d" % (int(nrows.max()), row_cap))
    out = np.zeros(nq, record_dtype(sd, row_cap))
    out["hdr"][:, 0], out["hdr"][:, 1], out["hdr"][:, 2] = counts[:, 1], counts[:, 0], nrows
    valid = np.arange(sd)[None, :] < counts[:, :1]
    out["w"] = np.where(valid, cand[:, :, 2], 0.0)
    out["id"] = np.where(valid, cand[:, :, 0], 0).astype(np.uint32)
    out["raw"] = np.where(valid, cand[:, :, 1], 0).astype(np.uint32)
    if len(rows):
        q = np.repeat(np.arange(nq), nrows)
        k = np.arange(len(rows)) - np.repeat(row_off[:-1], nrows)
        out["rows"][q, k] = rows
    return out


def merge_shard_batch(gathered: np.ndarray, search_depth: int = None, row_cap: int = None):
    """Vectorised merge_sharded_results over a whole batch.
    gathered: (S, nq) structured records of all shards.  Returns (rows (R,7) int32 in
    (query, global rank) order, row_off (nq+1)).

    No sort of the merged candidate lists: only ids that produced rows need a global rank, and
    the rank of id x is the number of published candidates that order before it by (weight desc,
    id desc) - found by one bisection per (row, shard) in that shard's already ordered list."""
    S, nq = gathered.shape
    sd = gathered.dtype["w"].shape[0]
    rcap = gathered.dtype["rows"].shape[0]
    depth = np.minimum(gathered["hdr"][:, :, 0].sum(axis=0), sd if search_depth is None else search_depth).astype(np.int64)
    ncand = gathered["hdr"][:, :, 1].astype(np.int64)                                         # (S, nq)
    nrows = gathered["hdr"][:, :, 2].astype(np.int64)
    W, I = gathered["w"], gathered["id"].astype(np.int64)                                      # (S, nq, sd)
    s_idx, q_idx, k_idx = np.nonzero(np.arange(rcap)[None, None, :] < nrows[:, :, None])
    if len(q_idx) == 0:
        return np.zeros((0, 7), np.int32), np.zeros(nq + 1, np.int64)
    r = gathered["rows"][s_idx, q_idx, k_idx].astype(np.int64)                                 # (R0, 7)
    w_x = W[s_idx, q_idx, r[:, 4]][:, None]          # column 4 = rank in the shard's own list
    i_x = r[:, :1]
    shard = np.arange(S)[None, :]
    lo = np.zeros((len(r), S), np.int64)
    hi = ncand[:, q_idx].T.copy()                                                             # (R0, S)
    for _ in range(int(sd).bit_length()):
        active = lo < hi
        mid = (lo + hi) >> 1
        at = np.minimum(mid, sd - 1)
        w = W[shard, q_idx[:, None], at]
        before = (w > w_x) | ((w == w_x) & (I[shard, q_idx[:, None], at] > i_x))
        lo = np.where(active & before, mid + 1, lo)
        hi = np.where(active & ~before, mid, hi)
    pos = lo.sum(axis=1)
    keep = pos < depth[q_idx]
    r, q_idx, pos, k_idx = r[keep], q_idx[keep], pos[keep], k_idx[keep]
    r[:, 4] = pos
    o = np.lexsort((k_idx, pos, q_idx))            # query, then global rank, then emission order
    r, q_idx = r[o], q_idx[o]
    off = np.zeros(nq + 1, np.int64)
    np.add.at(off, q_idx + 1, 1)
    return r.astype(np.int32), np.cumsum(off)


# ---- the product path: pack, all-gather and merge on the device -------------------------
def match_sharded_batch(matcher, ht, packed_queries, row_cap: int = 16, group=None, fetch: bool = True):
    """Sharded-table match of a packed (query rows, offsets) batch - every rank passes the same
    batch, its device table restricted to its id range.  On the device: probe + rank the shard
    (afp_match_batch, publish mode), pack one record per query (afp_shard_pack), ONE all-gather of
    the record buffers (torch.distributed: NCCL device-to-device; under gloo the bytes take the
    host route), merge (afp_shard_merge).  Returns (rows, offsets): the rows a single table gives,
    in candidate-rank order per query (what Matcher.match_batch(sort=False) returns); with
    fetch=False the result stays on the device (None, None)."""
    import ctypes as C
    import torch
    from . import _lib
    qrows, qoff = packed_queries
    if not hasattr(qrows, "data_ptr"):            # a torch CUDA tensor (int32 [R][2]) is used in place
        qrows = np.ascontiguousarray(qrows, dtype=np.int32).reshape(-1, 2)
    qoff = np.ascontiguousarray(qoff, dtype=np.int64)
    nq = len(qoff) - 1
    sd = max(int(matcher.search_depth), 1)
    p = matcher._params()
    p.publish_candidates = 1
    ctx = ht._sync_device()
    matcher._run(ctx, p, qrows, nq, qoff)
    rb = int(ctx.lib.afp_shard_record_bytes(sd, int(row_cap)))
    if rb < 0:
        raise ValueError("row_cap must be even and >= 2")
    dev = torch.device("cuda", ctx.device)
    mine = torch.empty((max(nq, 1), rb), dtype=torch.uint8, device=dev)
    try:
        ctx.check(ctx.lib.afp_shard_pack(ctx.h, int(row_cap), mine.data_ptr()))
    except _lib.AfpError as e:
        if "row capacity" in str(e):
            raise ValueError("a shard produced more than row_cap=%d rows for one query" % row_cap)
        raise
    rank, ws = world()
    if ws == 1:
        gathered = mine
    else:
        import torch.distributed as dist
        if dist.get_backend(group) == "nccl":
            gathered = torch.empty((ws * mine.shape[0], rb), dtype=torch.uint8, device=dev)
            dist.all_gather_into_tensor(gathered, mine, group=group)
        else:                                    # gloo: same bytes through host memory
            h = mine.cpu()
            g = torch.empty((ws * h.shape[0], rb), dtype=torch.uint8)
            dist.all_gather_into_tensor(g, h, group=group)
            gathered = g.to(dev)
        torch.cuda.current_stream(dev).synchronize()
    total = C.c_int64(0)
    ctx.check(ctx.lib.afp_shard_merge(ctx.h, gathered.data_ptr(), ws, nq, sd, int(row_cap), C.byref(total)))
    if not fetch:
        return None, None
    rows = np.empty((int(total.value), 7), np.int32)
    roff = np.zeros(nq + 1, np.int64)
    ctx.check(ctx.lib.afp_fetch_match_rows(ctx.h, rows.ctypes.data if len(rows) else None, 1,
                                           roff.ctypes.data_as(C.POINTER(C.c_int64))))
    return rows, roff
