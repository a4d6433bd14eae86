"""Multi-GPU plumbing: one process per GPU, `torch.distributed` for the rendezvous.

The reference's only parallelism is sharding the FILE LIST over OS processes
(`multiproc_add`, audfprint.py:199-235: file ix goes to process ix % ncores) and
pickling results back.  The same shape is used here:

* fingerprinting: file i -> rank i % world; NO data-path collective (results are
  per-file and gathered as host objects only if the caller asks for them);
* building ONE table from a multi-GPU ingest (`ingest_sharded`, the reference's
  `new` / `add --ncores N`): every rank stores its own files into a fresh table on
  its GPU, the root receives the tables in rank order (NCCL device to device) and
  merges each into its table on the device, as `multiproc_add` merges its workers'
  tables;
* matching, table replicated (419 MB << 80 GB): query j -> rank j % world; no
  data-path collective (`match_files_sharded`, the reference's `match --ncores N`);
* matching, table sharded by track-id range (SURVEY.md §8e, BASELINE configs[4]):
  every rank sees every query, computes the candidate list and result rows of
  ITS ids, and ONE all-gather of fixed-size per-query records merges them:
  `merge_sharded_results` below is exact because an id inside the global top-D
  (D = min(sum n_above, search_depth)) is inside its own shard's local top-D.
  With exact_count / find_time_range one all-reduce (MAX) of each query's largest
  query time comes first, so that every shard packs its (qtime, hash) keys with the
  whole table's key width; see match_sharded_batch.

Nothing here computes on the CPU; it only moves tables and small result records.
"""
from __future__ import annotations

import numpy as np


def world(group=None):
    """(rank, world_size) in `group` (None: the default process group), (0, 1) when torch.distributed
    is not initialised."""
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return dist.get_rank(group), dist.get_world_size(group)
    except ImportError:
        pass
    return 0, 1


def _collective_device(group, device=None):
    """Where the buffers of a collective over `group` live: CUDA device `device` (None: torch's current
    one) under NCCL, host memory under gloo, which the device data reaches by a round trip."""
    import torch
    import torch.distributed as dist
    if dist.get_backend(group) != "nccl":
        return torch.device("cpu")
    return torch.device("cuda", torch.cuda.current_device() if device is None else device)


def _global_rank(group, r):
    import torch.distributed as dist
    return r if group is None else dist.get_global_rank(group, r)


def _check_root(root, group):
    rank, ws = world(group)
    if not 0 <= int(root) < ws:
        raise ValueError("root %d outside the group's %d ranks" % (int(root), ws))


# status of one rank's part of an entry point, exchanged before any result moves
_OK, _IO_ERROR, _FAILED = 0, 1, 2


def _status_code(err, io_errors_everywhere=True):
    """This rank's status: _OK without an exception, _IO_ERROR for an IOError that every rank is to
    raise (with io_errors_everywhere), _FAILED otherwise."""
    if err is None:
        return _OK
    return _IO_ERROR if io_errors_everywhere and isinstance(err, IOError) else _FAILED


def _raise_if_failed(err, codes, what, group=None):
    """Raise the same thing on every rank of `group` when one failed; `err` is this rank's exception
    (or None) and `codes` the _status_code of every rank, in rank order, gathered by the caller.  The
    messages are gathered only when a rank failed, by every rank.  The failing rank raises its own
    exception; the others raise the first failing rank's IOError when its code is _IO_ERROR, else a
    RuntimeError naming `what`, that rank and its message."""
    failed = [r for r, c in enumerate(codes) if int(c) != _OK]
    if not failed:
        return
    msgs = gather_objects("" if err is None else str(err), group)
    if err is not None:
        raise err
    r = failed[0]
    if int(codes[r]) == _IO_ERROR:
        raise IOError(msgs[r])
    raise RuntimeError("%s: rank %d failed: %s" % (what, r, msgs[r]))


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
    rank, ws = world(group)
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


def _allgather_bytes(mine: np.ndarray, group=None, device=None) -> np.ndarray:
    """all_gather of one 1-D array per rank (a structured one included), with buffers where
    _collective_device puts them -> (world, len) array."""
    rank, ws = world(group)
    if ws == 1:
        return mine[None]
    import torch
    import torch.distributed as dist
    dev = _collective_device(group, device)
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
    below is the throughput path).  With exact_count or find_time_range set the queries go through
    match_sharded_batch, which finishes them on the device."""
    if matcher.exact_count or matcher.find_time_range:
        from ._lib import pack_rows
        packed, qoff = pack_rows(queries)
        rows, roff = match_sharded_batch(matcher, ht, (packed, qoff), row_cap, group)
        return [r[(-r[:, 1]).argsort(), ] for r in (rows[roff[i]:roff[i + 1]] for i in range(len(qoff) - 1))]
    mine = matcher.match_batch_shard(ht, queries)
    shards = allgather_shard_records(mine, matcher.search_depth, row_cap, group)
    out = []
    for qi in range(len(queries)):
        rows = merge_sharded_results([s[qi] for s in shards], matcher.search_depth)
        out.append(rows[(-rows[:, 1]).argsort(), ])          # audfprint_match.py:335
    return out


# ---- vectorised host statement of pack / merge (tests; checks the device kernels) --------
STATUS_OVERFLOW = 1        # status word (hdr[3]) after an options finish: bit 0 = more rows than row_cap,
                           # bits 1-30 = 1 + the smallest local rank whose quantile read failed


def pack_shard_batch(cand, counts, rows, row_off, row_cap: int, fail_rank=None) -> np.ndarray:
    """The wire records built without a Python loop from what afp_fetch_match_candidates /
    afp_fetch_match_rows return: cand (nq, sd, 3) f64, counts (nq, 2) i32 [entries, n_above],
    rows (R, 7) i32, row_off (nq+1).

    fail_rank (nq,) int, -1 = none: the records of an options finish on a shard (what
    afp_shard_pack writes after afp_match_options_shard_finish).  Then nothing raises: the status
    word carries the smallest local rank whose quantile read failed and the overflow bit, nrows is
    the number of rows the shard produced and the record holds the first row_cap of them."""
    nq, sd = cand.shape[0], cand.shape[1]
    nrows = np.diff(row_off)
    if fail_rank is None and nq and nrows.max(initial=0) > row_cap:
        raise ValueError("a shard produced %d rows for one query, row_cap is %d" % (int(nrows.max()), row_cap))
    out = np.zeros(nq, record_dtype(sd, row_cap))
    out["hdr"][:, 0], out["hdr"][:, 1], out["hdr"][:, 2] = counts[:, 1], counts[:, 0], nrows
    if fail_rank is not None:
        fail_rank = np.asarray(fail_rank, np.int64)
        out["hdr"][:, 3] = np.where(nrows > row_cap, STATUS_OVERFLOW, 0) | np.where(fail_rank >= 0, (fail_rank + 1) << 1, 0)
    valid = np.arange(sd)[None, :] < counts[:, :1]
    out["w"] = np.where(valid, cand[:, :, 2], 0.0)
    out["id"] = np.where(valid, cand[:, :, 0], 0).astype(np.uint32)
    out["raw"] = np.where(valid, cand[:, :, 1], 0).astype(np.uint32)
    if len(rows):
        q = np.repeat(np.arange(nq), nrows)
        k = np.arange(len(rows)) - np.repeat(row_off[:-1], nrows)
        held = k < row_cap
        out["rows"][q[held], k[held]] = rows[held]
    return out


def _global_ranks(W, I, ncand, s_idx, q_idx, lr):
    """Global rank of local rank lr of shard s_idx for query q_idx: the number of published
    candidates of all shards that order before it by (weight desc, id desc) - one bisection per
    shard in that shard's already ordered list (in its own shard that number is lr)."""
    S, sd = W.shape[0], W.shape[2]
    w_x = W[s_idx, q_idx, lr][:, None]
    i_x = I[s_idx, q_idx, lr][:, None]
    shard = np.arange(S)[None, :]
    lo = np.zeros((len(lr), S), np.int64)
    hi = ncand[:, q_idx].T.copy()                                                             # (n, S)
    for _ in range(int(sd).bit_length()):
        active = lo < hi
        mid = (lo + hi) >> 1
        at = np.minimum(mid, sd - 1)
        w = W[shard, q_idx[:, None], at]
        before = (w > w_x) | ((w == w_x) & (I[shard, q_idx[:, None], at] > i_x))
        lo = np.where(active & before, mid + 1, lo)
        hi = np.where(active & ~before, mid, hi)
    return lo.sum(axis=1)


def check_shard_status(gathered: np.ndarray, search_depth: int = None):
    """The merge's reading of the status words of all shards' records (afp_shard_merge): IndexError
    if a failed quantile read lies at a global rank < D (the single table reaches that candidate
    too), else ValueError naming the largest row count of an overflowed record."""
    st = gathered["hdr"][:, :, 3].astype(np.int64)
    if not st.any():
        return
    sd = gathered.dtype["w"].shape[0]
    depth = np.minimum(gathered["hdr"][:, :, 0].sum(axis=0), sd if search_depth is None else search_depth)
    s_idx, q_idx = np.nonzero((st >> 1) > 0)
    if len(s_idx):
        g = _global_ranks(gathered["w"], gathered["id"].astype(np.int64), gathered["hdr"][:, :, 1].astype(np.int64),
                          s_idx, q_idx, (st[s_idx, q_idx] >> 1) - 1)
        if np.any(g < depth[q_idx]):
            raise IndexError("time_quantile index outside a support (IndexError)")
    over = (st & STATUS_OVERFLOW) != 0
    if over.any():
        raise ValueError("row capacity: a shard produced %d rows for one query, row_cap is %d"
                         % (int(gathered["hdr"][:, :, 2][over].max()), gathered.dtype["rows"].shape[0]))


def merge_shard_batch(gathered: np.ndarray, search_depth: int = None, row_cap: int = None):
    """Vectorised merge_sharded_results over a whole batch.
    gathered: (S, nq) structured records of all shards.  Returns (rows (R,7) int32 in
    (query, global rank) order, row_off (nq+1)).

    No sort of the merged candidate lists: only ids that produced rows need a global rank, and
    the rank of id x is the number of published candidates that order before it by (weight desc,
    id desc) - found by one bisection per (row, shard) in that shard's already ordered list."""
    check_shard_status(gathered, search_depth)
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
    pos = _global_ranks(W, I, ncand, s_idx, q_idx, r[:, 4])      # column 4 = rank in the shard's own list
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
    fetch=False the result stays on the device (None, None).

    With matcher.exact_count / find_time_range (time_quantile) the shard is finished before the
    pack, in two calls around one all-reduce (MAX) of one int32 per query - the query's largest
    qtime, which sets the width of the (qtime, hash) keys the exact count compares
    (audfprint_match.py:157-167) and must be the whole table's: afp_match_options_shard_rank,
    the all-reduce (NCCL in place; gloo through host memory), afp_match_options_shard_finish.
    Nothing data-dependent raises between the collectives; the merge raises the same error on every
    rank: IndexError when a quantile index leaves its support at a candidate the single table
    finishes, ValueError when a shard produced more than row_cap rows for a query."""
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
    options = bool(matcher.exact_count or matcher.find_time_range)
    rb = int(ctx.lib.afp_shard_record_bytes(sd, int(row_cap)))
    if rb < 0:
        raise ValueError("row_cap must be even and >= 2")
    dev = torch.device("cuda", ctx.device)
    rank, ws = world(group)
    if not options:
        matcher._run(ctx, p, qrows, nq, qoff)
    else:
        qmax = torch.empty(max(nq, 1), dtype=torch.int32, device=dev)      # written by the ranking call
        matcher._run(ctx, p, qrows, nq, qoff, (matcher.exact_count, matcher.find_time_range, matcher.time_quantile),
                     shard_qmax=qmax)
        if ws > 1:
            import torch.distributed as dist
            buf = qmax.to(_collective_device(group, ctx.device))         # in place under NCCL
            dist.all_reduce(buf, op=dist.ReduceOp.MAX, group=group)
            if buf is not qmax:
                qmax.copy_(buf)
        with ctx.after_torch(qmax):
            ctx.check(ctx.lib.afp_match_options_shard_finish(ctx.h, C.c_void_p(qmax.data_ptr()), None))
    mine = torch.empty((max(nq, 1), rb), dtype=torch.uint8, device=dev)
    try:
        with ctx.after_torch(mine):               # torch's pending reads of its memory come first
            ctx.check(ctx.lib.afp_shard_pack(ctx.h, int(row_cap), mine.data_ptr()))
    except _lib.AfpError as e:
        if "row capacity" in str(e):
            raise ValueError("a shard produced more than row_cap=%d rows for one query" % row_cap)
        raise
    if ws == 1:
        gathered = mine
    else:
        import torch.distributed as dist
        cdev = _collective_device(group, ctx.device)
        g = torch.empty((ws * mine.shape[0], rb), dtype=torch.uint8, device=cdev)
        dist.all_gather_into_tensor(g, mine.to(cdev), group=group)
        gathered = g.to(dev)
    total = C.c_int64(0)
    with ctx.after_torch(gathered):
        ctx.check(ctx.lib.afp_shard_merge(ctx.h, gathered.data_ptr(), ws, nq, sd, int(row_cap), C.byref(total)))
    if not fetch:
        return None, None
    return matcher._fetch_rows(ctx, int(total.value), nq)


# ---- one table from a multi-GPU ingest (the reference's multiproc_add) --------------------
def ingest_sharded(analyzer, ht, names, signals, root=0, replicate=False, report=None, group=None):
    """`audfprint.py new / add --ncores N` (multiproc_add, audfprint.py:199-235) over the ranks of
    a process group, one GPU each.  `names` / `signals` are this rank's own files, dealt as the
    reference deals them (shard_indices: file i -> rank i % world).

    1. The rank ingests its files into a fresh table of ht's geometry on its GPU
       (Analyzer.ingest_batch), drawing from this process's `random` state; the reference's worker r
       draws from its own, so seed each rank's `random` (e.g. random.seed(1000 + rank)).
    2. One all-gather of a status word, the rank's name and hash counts and the root's base name
       count and geometry.  If any rank's ingest raised, every rank raises before any table moves:
       the failing rank its own exception, the others a RuntimeError naming the first failing rank.
       Geometries that disagree raise ValueError, and a merged id that would not fit in
       32 - maxtimebits bits raises OverflowError, on every rank alike.
    3. The rank's table is exported on its device (HashTable.export_device).  The root receives the
       tables in rank order - NCCL send / recv device to device, or through host memory under gloo -
       and merges them into `ht` with ONE merge_batch, in rank order, its own table included (the
       merge of an empty table is not the table itself: counts above depth become depth).  The root's
       own table never goes through the host.
    4. Names and hashesperid travel as host objects.  The merged names are rank-major:
       ht.names + names of rank 0 + names of rank 1 + ...
    5. `report`, on the root, receives the reference's line "hash_table r has N files H hashes" for
       each rank r, in rank order, as a one-line list.
    6. With replicate=True the root exports the merged table and broadcasts it; every rank installs it
       as its device copy (afp_table_upload from device memory) with the same names and hashesperid.
       Otherwise the other ranks' `ht` are unchanged.  np.random advances on the root only.
    Returns the number of hashes stored for each of this rank's files."""
    _check_root(root, group)
    if len(names) != len(signals):
        raise ValueError("%d names for %d signals" % (len(names), len(signals)))
    return _ingest_and_merge(lambda local: analyzer.ingest_batch(local, list(names), list(signals)), ht, int(root),
                             replicate, report, group, False)


def _ingest_and_merge(ingest, ht, root, replicate, report, group, io_errors_everywhere):
    """Steps 1-6 of ingest_sharded, with step 1 as `ingest(local_table)` -> this rank's result.  With
    io_errors_everywhere an IOError raised by one rank's ingest is raised, with its message, on every
    rank (an unreadable file under fail_on_error); otherwise the others raise a RuntimeError."""
    import torch
    from . import _lib
    from .hash_table import DeviceTable, HashTable
    rank, ws = world(group)
    ctx = _lib.context(ht.device)
    dev = torch.device("cuda", ctx.device)
    if ws > 1:
        import torch.distributed as dist
        cdev = _collective_device(group, ctx.device)
    hb, depth, mtb = int(ht.hashbits), int(ht.depth), int(ht.maxtimebits)

    # 1. this rank's files into a fresh table
    local = HashTable(hashbits=hb, depth=depth, maxtime=1 << mtb, device=ht.device)
    err, mine, counts = None, None, []
    try:
        counts = ingest(local)
        mine = local.export_device()
    except Exception as e:          # raised on every rank after the all-gather
        err = e
    local._disown_device()          # its rows live on in `mine`: no pull to the host when `ht` takes the device
    del local
    nhashes = int(mine.counts.sum(dtype=torch.int64)) if mine is not None else 0

    # 2. status, name and hash counts, the root's base and geometry, from every rank
    info = np.array([_status_code(err, io_errors_everywhere), len(mine.names) if mine is not None else 0, nhashes,
                     len(ht.names), hb, depth, mtb], np.int64)
    infos = _allgather_bytes(info, group, ctx.device)
    _raise_if_failed(err, infos[:, 0], "ingest_sharded", group)
    if (infos[:, 4:] != infos[root, 4:]).any():
        raise ValueError("ingest_sharded: the ranks' tables disagree on hashbits / depth / maxtimebits")
    nn = int(infos[root, 3])
    for r in range(ws):
        if nn << mtb >= 1 << 32:
            raise OverflowError("id offset %d does not fit in %d id bits" % (nn, 32 - mtb))
        nn += int(infos[r, 1])
        if infos[r, 1] and (nn + 1) << mtb > 1 << 32:
            raise OverflowError("id %d does not fit in %d id bits" % (nn - 1, 32 - mtb))

    # 3. + 4. the tables to the root in rank order, names and hashesperid as host objects
    nb = 1 << hb
    book = [(mine.names, mine.hashesperid)]
    if ws > 1:
        book = [None] * ws if rank == root else None
        dist.gather_object((mine.names, mine.hashesperid), book, dst=_global_rank(group, root), group=group)
    if rank == root:
        tables = []
        for r in range(ws):
            if r == rank:
                tables.append(mine)
                continue
            tab = torch.empty((nb, depth), dtype=torch.int32, device=cdev)
            cnt = torch.empty(nb, dtype=torch.int32, device=cdev)
            dist.recv(tab, src=_global_rank(group, r), group=group)
            dist.recv(cnt, src=_global_rank(group, r), group=group)
            tables.append(DeviceTable(tab.to(dev), cnt.to(dev), book[r][0], book[r][1], hb, depth, mtb))
        if report is not None:
            for r in range(ws):
                report(["hash_table %d has %d files %d hashes" % (r, int(infos[r, 1]), int(infos[r, 2]))])
        ht.merge_batch(tables)
        del tables
    else:
        dst = _global_rank(group, root)
        dist.send(mine.table.to(cdev), dst=dst, group=group)
        dist.send(mine.counts.to(cdev), dst=dst, group=group)
    del mine

    # 6. the merged table to every rank
    if replicate and ws > 1:
        src = _global_rank(group, root)
        if rank == root:
            snap = ht.export_device()
            obj = [(snap.names, snap.hashesperid)]
            tab, cnt = snap.table.to(cdev), snap.counts.to(cdev)
        else:
            obj = [None]
            tab = torch.empty((nb, depth), dtype=torch.int32, device=cdev)
            cnt = torch.empty(nb, dtype=torch.int32, device=cdev)
        dist.broadcast_object_list(obj, src=src, group=group)
        dist.broadcast(tab, src=src, group=group)
        dist.broadcast(cnt, src=src, group=group)
        if rank != root:
            ht._install_device(DeviceTable(tab.to(dev), cnt.to(dev), obj[0][0], obj[0][1], hb, depth, mtb))
    return counts


# ---- matching a list of files against a replicated table (the reference's match --ncores N) ----
def gather_in_list_order(mine, n, root=0, group=None):
    """Rank r's results of items r, r + world, r + 2 world, ... (shard_indices) -> the whole list of
    n results in list order on the root, None on the other ranks: one gather_object."""
    rank, ws = world(group)
    return _gather_by_index(shard_indices(n, rank, ws), mine, n, root, group)


def _gather_by_index(idx, mine, n, root, group):
    """This rank's results `mine` of the list positions `idx` -> the whole list of n results on the
    root, None on the other ranks: one gather_object."""
    rank, ws = world(group)
    if ws == 1:
        return list(mine)
    import torch.distributed as dist
    book = [None] * ws if rank == root else None
    dist.gather_object((np.asarray(idx).tolist(), list(mine)), book, dst=_global_rank(group, root), group=group)
    if rank != root:
        return None
    out = [None] * n
    for ids, results in book:
        for i, m in zip(ids, results):
            out[i] = m
    return out


def match_files_sharded(matcher, analyzer, ht, filenames, root=0, group=None):
    """`audfprint.py match --ncores N` (audfprint.py:257-267) over the ranks of a process group, one
    GPU each, with the same table on every rank (e.g. ingest_sharded(replicate=True), or one database
    loaded by every rank).  Every rank passes the whole list.

    1. One all-gather of every rank's table geometry (hashbits, depth, maxtimebits) and name count;
       a mismatch raises ValueError on every rank before any file is read.
    2. File j goes to rank j % world (shard_indices).  Each rank runs Matcher.files_match_to_msgs on
       its files, numbering file j as j, and its analyzer counts its own files.
    3. One all-gather of a status word.  If a rank failed, every rank raises: the same IOError when
       the failure was an unreadable file (analyzer.fail_on_error), otherwise the failing rank its
       own exception and the others a RuntimeError naming it.  No rank is left in a collective.
    4. The root returns the message lists in list order, as joblib returns them; the other ranks
       return None."""
    from . import _lib
    _check_root(root, group)
    rank, ws = world(group)
    n = len(filenames)
    info = np.array([int(ht.hashbits), int(ht.depth), int(ht.maxtimebits), len(ht.names)], np.int64)
    infos = _allgather_bytes(info, group, _lib.context(ht.device).device if ws > 1 else None)
    if (infos != infos[0]).any():
        raise ValueError("match_files_sharded: the ranks' tables disagree on hashbits / depth / maxtimebits / "
                         "number of names: %s" % infos.tolist())
    idx = shard_indices(n, rank, ws)
    err, mine = None, []
    try:
        mine = analyzer._list_form(lambda: matcher._files_msgs(analyzer, ht, [filenames[i] for i in idx],
                                                               [int(i) for i in idx]))
    except Exception as e:          # raised on every rank after the status exchange
        err = e
    _raise_if_failed(err, gather_objects(_status_code(err), group), "match_files_sharded", group)
    return _gather_by_index(idx, mine, n, int(root), group)


# ---- new / add and precompute from a list of files (the reference's --ncores N) ----------------
def ingest_files_sharded(analyzer, ht, filenames, root=0, replicate=False, report=None, group=None):
    """`audfprint.py new / add --ncores N` from files: ingest_sharded with every rank reading its own
    files.  Every rank passes the whole list and takes file j when j % world is its rank
    (shard_indices, as multiproc_add deals), then runs Analyzer.ingest_files into a fresh table;
    the status exchange, the tables' trip to the root, the one merge_batch, the report lines and
    the optional replication are ingest_sharded's.  An unreadable file (fail_on_error) raises the
    same IOError on every rank.  Returns ingest_files' (duration, hashes) of this rank's files."""
    _check_root(root, group)
    rank, ws = world(group)
    idx = shard_indices(len(filenames), rank, ws)
    mine = [filenames[i] for i in idx]
    return _ingest_and_merge(lambda local: analyzer.ingest_files(local, mine), ht, int(root), replicate, report,
                             group, True)


def precompute_owners(opnames, world_size: int) -> np.ndarray:
    """Rank that precomputes each file of a list whose output names are `opnames`: the rank of the
    FIRST file naming that output (j % world), so that every file writing one output runs on one
    rank in list order and the list-order effects of skip_existing and overwriting hold."""
    first = {}
    owners = np.empty(len(opnames), np.int64)
    for j, name in enumerate(opnames):
        owners[j] = first.setdefault(name, j % world_size)
    return owners


def precompute_files_sharded(analyzer, filenames, precompdir, type='hashes', skip_existing=False,
                             strip_prefix=None, root=0, group=None):
    """`audfprint.py precompute --ncores N` over the ranks of a process group, one GPU each.  Every
    rank passes the whole list and runs Analyzer.precompute_files on the files it owns
    (precompute_owners), in list order.  Failures are handled as in match_files_sharded: the same
    IOError on every rank for an unreadable file, otherwise the failing rank's own exception and a
    RuntimeError on the others.  The root returns one message list per file in list order; the other
    ranks return None."""
    from .analyzer import precompute_name
    _check_root(root, group)
    rank, ws = world(group)
    opnames = [precompute_name(f, precompdir, type == 'hashes', strip_prefix) for f in filenames]
    idx = np.flatnonzero(precompute_owners(opnames, ws) == rank)
    err, mine = None, []
    try:
        mine = analyzer.precompute_files([filenames[i] for i in idx], precompdir, type, skip_existing, strip_prefix)
    except Exception as e:          # raised on every rank after the status exchange
        err = e
    _raise_if_failed(err, gather_objects(_status_code(err), group), "precompute_files_sharded", group)
    return _gather_by_index(idx, mine, len(filenames), int(root), group)
