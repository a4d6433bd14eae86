// HashTable.store on the device-resident table, batched over the files of an ingest
// (SURVEY.md §8f-1; reference hash_table.py:91-138).
//
// Reference semantics, per (time, hash) row of a track, IN SEQUENCE (files in call order, rows
// in their (time, hash) order):
//     count = counts[hash]
//     if count < depth:  table[hash][count] = val            val = ((id + 1) << maxtimebits) + (time & mask)
//     else:              slot = random.randint(0, count); if slot < depth: table[hash][slot] = val
//     counts[hash] = count + 1
// An entry's slot therefore is counts0[bucket] + (number of EARLIER entries of the batch in the
// same bucket) - a rank inside the bucket by sequence number - and everything that lands below
// `depth` can be written in parallel.  The device does exactly that:
//   1. per entry: bucket, value; histogram of the batch over the buckets (global atomics,
//      order-free);
//   2. exclusive scan of the histogram -> one segment per bucket; the entries' sequence numbers
//      are scattered into their segments (arrival order is arbitrary) ...
//   3. ... and every segment is put in sequence order (a handful of entries: one thread; the few
//      hot buckets: one CTA ranking by counting), which gives each entry its slot;
//   4. entries whose slot is >= depth are the overflow: they are compacted IN SEQUENCE ORDER and
//      handed to the host, which replays the reference's random.randint draws on them (a C
//      implementation of CPython's MT19937 / _randbelow, afp_mt_randint_replay below) and sends
//      back the resulting (bucket, slot, value) patches.
// With the same RNG state the device table is therefore bit-identical to what the reference's
// store() builds (tests/test_gpu_store.py, against the reference-pinned host store();
// tests/test_gpu_table_edges.py, against the sequential statement of tests/table_reference.py at
// the LIGHT / SCAP / SB edges, the scan carry, the masks and the last-writer scratch).
#include <algorithm>
#include "afp_internal.cuh"

namespace {

struct StoreArgs {
  const int32_t* rows;       // [M][2] (time, hash), CSR by file
  const int64_t* row_off;    // [nfiles+1]
  const int64_t* ids;        // [nfiles] track id of every file
  int nfiles;
  int hashbits, depth, mtb;
  uint32_t* table;
  int32_t* counts;
  uint32_t* eval;            // [M] value of every entry
  uint32_t* cnt_new;         // [nb] entries of the batch per bucket; later the scatter cursor
  const int64_t* seg_off;    // [nb+1]
  int32_t* seq;              // [M] entry numbers grouped by bucket
  int32_t* ovf_pos;          // [M] count-before of overflowing entries, -1 otherwise
  int32_t* heavy;            // list of buckets with more than LIGHT entries
  int* nheavy;
};

constexpr int LIGHT = 16;

__device__ __forceinline__ uint32_t bucket_of(const StoreArgs& a, int64_t i) {
  return (uint32_t)a.rows[2 * i + 1] & ((1u << a.hashbits) - 1u);
}

// one CTA per file: entry values + bucket histogram
__global__ void __launch_bounds__(256) afp_store_count_kernel(StoreArgs a) {
  const int f = blockIdx.x;
  const int64_t r0 = a.row_off[f], r1 = a.row_off[f + 1];
  const uint32_t idval = (uint32_t)((a.ids[f] + 1) << a.mtb);
  const uint32_t tmask = (1u << a.mtb) - 1u;
  for (int64_t i = r0 + threadIdx.x; i < r1; i += blockDim.x) {
    a.eval[i] = idval + ((uint32_t)a.rows[2 * i] & tmask);
    a.ovf_pos[i] = -1;
    atomicAdd(&a.cnt_new[bucket_of(a, i)], 1u);
  }
}

__global__ void afp_store_scatter_kernel(StoreArgs a, int64_t M, uint32_t* cursor) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const uint32_t b = bucket_of(a, i);
  a.seq[a.seg_off[b] + atomicAdd(&cursor[b], 1u)] = (int32_t)i;
}

__device__ __forceinline__ void place(const StoreArgs& a, uint32_t b, int c0, int rank, int32_t i) {
  const int pos = c0 + rank;
  if (pos < a.depth) a.table[(size_t)b * a.depth + pos] = a.eval[i];
  else a.ovf_pos[i] = pos;             // the reference draws randint(0, pos) for this one
}

// one thread per bucket: sort the bucket's (few) entries by sequence number, place them
__global__ void afp_store_place_kernel(StoreArgs a, int64_t nb) {
  const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb) return;
  const int64_t s0 = a.seg_off[b];
  const int n = (int)(a.seg_off[b + 1] - s0);
  if (n == 0) return;
  if (n > LIGHT) {
    a.heavy[atomicAdd(a.nheavy, 1)] = (int32_t)b;
    return;
  }
  int32_t e[LIGHT];
#pragma unroll
  for (int k = 0; k < LIGHT; ++k) e[k] = k < n ? a.seq[s0 + k] : 0x7fffffff;
  const int c0 = a.counts[b];
#pragma unroll
  for (int k = 0; k < LIGHT; ++k)
    if (k < n) {                          // rank = number of smaller sequence numbers (all distinct)
      int r = 0;
#pragma unroll
      for (int j = 0; j < LIGHT; ++j) r += e[j] < e[k] ? 1 : 0;
      place(a, (uint32_t)b, c0, r, e[k]);
    }
  a.counts[b] = c0 + n;
}

// one CTA per hot bucket: rank = number of smaller sequence numbers in the segment
__global__ void __launch_bounds__(256) afp_store_heavy_kernel(StoreArgs a) {
  extern __shared__ int32_t s_seq[];
  constexpr int SCAP = 8192;
  const uint32_t b = (uint32_t)a.heavy[blockIdx.x];
  const int64_t s0 = a.seg_off[b];
  const int n = (int)(a.seg_off[b + 1] - s0);
  const int32_t* src = a.seq + s0;
  const bool in_smem = n <= SCAP;
  if (in_smem) {
    for (int k = threadIdx.x; k < n; k += blockDim.x) s_seq[k] = src[k];
    __syncthreads();
    src = s_seq;
  }
  const int c0 = a.counts[b];
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const int32_t x = src[k];
    int r = 0;
    for (int j = 0; j < n; ++j) r += src[j] < x ? 1 : 0;
    place(a, b, c0, r, x);
  }
  __syncthreads();
  if (threadIdx.x == 0) a.counts[b] = c0 + n;
}

// ---- a scan that scales: block sums -> scan of the sums -> per-block scan with carry ----
constexpr int SB = 1024;
__global__ void __launch_bounds__(SB) afp_flag_blocksum_kernel(const int32_t* ovf_pos, int64_t M, int32_t* part) {
  __shared__ int s[SB / 32];
  const int64_t i = (int64_t)blockIdx.x * SB + threadIdx.x;
  int v = (i < M && ovf_pos[i] >= 0) ? 1 : 0;
  v = __reduce_add_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < SB / 32; ++w) t += s[w];
    part[blockIdx.x] = t;
  }
}
// overflow entries, compacted in sequence order: (bucket, count-before, value)
__global__ void __launch_bounds__(SB) afp_ovf_compact_kernel(StoreArgs a, int64_t M, const int64_t* part_off,
                                                              uint32_t* o_bucket, int32_t* o_pos, uint32_t* o_val) {
  __shared__ int s[SB / 32];
  const int64_t i = (int64_t)blockIdx.x * SB + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int pos = i < M ? a.ovf_pos[i] : -1;
  const unsigned m = __ballot_sync(0xffffffffu, pos >= 0);
  if (lane == 0) s[warp] = __popc(m);
  __syncthreads();
  if (warp == 0) {
    int v = s[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += t;
    }
    s[lane] = v;
  }
  __syncthreads();
  if (pos >= 0) {
    const int64_t o = part_off[blockIdx.x] + (warp ? s[warp - 1] : 0) + __popc(m & ((1u << lane) - 1u));
    o_bucket[o] = bucket_of(a, i);
    o_pos[o] = pos;
    o_val[o] = a.eval[i];
  }
}

// The host returns ONE int per overflow entry: the slot random.randint drew (>= depth: no write).
// Several entries may name the same (bucket, slot); the sequential loop of the reference lets the
// LAST one win.  `last` is a table-sized scratch of entry numbers (zero between calls):
// pass A records the highest entry number per slot, pass B lets that entry write and clears.
__global__ void afp_slots_mark_kernel(const uint32_t* bucket, const int32_t* slot, int64_t n, int depth, uint32_t* last) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = slot[i];
  if (s >= 0 && s < depth) atomicMax(&last[(size_t)bucket[i] * depth + s], (uint32_t)(i + 1));
}
__global__ void afp_slots_write_kernel(const uint32_t* bucket, const int32_t* slot, const uint32_t* val, int64_t n,
                                       int depth, uint32_t* last, uint32_t* table) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = slot[i];
  if (s < 0 || s >= depth) return;
  const size_t k = (size_t)bucket[i] * depth + s;
  if (last[k] == (uint32_t)(i + 1)) {
    table[k] = val[i];
    last[k] = 0u;                       // only the winner clears: the scratch is all-zero again
  }
}

__global__ void afp_patch_kernel(uint32_t* table, int depth, const uint32_t* bucket, const int32_t* slot,
                                 const uint32_t* val, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) table[(size_t)bucket[i] * depth + slot[i]] = val[i];
}

}  // namespace

extern "C" {

int afp_table_create(afp_ctx* c, int32_t hashbits, int32_t depth, int32_t maxtimebits) {
  if (!c) return AFP_ERR_INVALID;
  if (hashbits < 1 || hashbits > 28 || depth < 1 || maxtimebits < 1 || maxtimebits > 24)
    AFP_FAIL(c, AFP_ERR_INVALID, "bad table geometry");
  AFP_CUDA(c, cudaSetDevice(c->device));
  const size_t nb = (size_t)1 << hashbits;
  c->tab.loaded = false;
  AFP_CUDA(c, c->tab.table.reserve(nb * (size_t)depth * sizeof(uint32_t)));
  AFP_CUDA(c, c->tab.counts.reserve(nb * sizeof(int32_t)));
  AFP_CUDA(c, c->tab.hashesperid.reserve(sizeof(uint32_t)));
  AFP_CUDA(c, cudaMemsetAsync(c->tab.table.p, 0, nb * (size_t)depth * sizeof(uint32_t), c->stream));
  AFP_CUDA(c, cudaMemsetAsync(c->tab.counts.p, 0, nb * sizeof(int32_t), c->stream));
  c->tab.hashbits = hashbits;
  c->tab.depth = depth;
  c->tab.maxtimebits = maxtimebits;
  c->tab.nids = 0;
  c->tab.hmin = 0;
  c->tab.loaded = true;
  return AFP_OK;
}

int afp_table_set_hashesperid(afp_ctx* c, const uint32_t* hashesperid, int64_t nids) {
  if (!c || nids < 0 || (nids > 0 && !hashesperid)) return AFP_ERR_INVALID;
  if (!c->tab.loaded) AFP_FAIL(c, AFP_ERR_STATE, "no table on the device");
  AFP_CUDA(c, cudaSetDevice(c->device));
  // a grown array may move: the previous one may still be read by kernels in flight
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  AFP_CUDA(c, c->tab.hashesperid.reserve(((size_t)nids + 1) * sizeof(uint32_t)));
  if (nids > 0)
    AFP_CUDA(c, cudaMemcpyAsync(c->tab.hashesperid.p, hashesperid, (size_t)nids * sizeof(uint32_t),
                                cudaMemcpyHostToDevice, c->stream));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  c->tab.nids = nids;
  return afp_table_stats(c);
}

int afp_table_store_batch(afp_ctx* c, const int32_t* rows, int rows_on_host, const int64_t* row_offsets,
                          int32_t nfiles, const int64_t* ids, int64_t* noverflow) {
  if (!c || nfiles < 0 || (nfiles > 0 && !ids)) return AFP_ERR_INVALID;
  if (!c->tab.loaded) AFP_FAIL(c, AFP_ERR_STATE, "no table on the device (afp_table_upload / afp_table_create)");
  AFP_CUDA(c, cudaSetDevice(c->device));
  c->store_novf = 0;
  if (noverflow) *noverflow = 0;
  if (nfiles == 0) return AFP_OK;
  const int32_t* drows = nullptr;
  const int64_t* droff = nullptr;
  int64_t M = 0;
  if (!rows) {                               // the hashes of the last fingerprint batch, in place
    if (!c->batch_valid) AFP_FAIL(c, AFP_ERR_STATE, "no fingerprint batch in the workspace");
    if (nfiles != c->nfiles) AFP_FAIL(c, AFP_ERR_INVALID, "nfiles differs from the fingerprint batch");
    int rc;
    if (c->total_hashes < 0 &&
        (rc = afp_read_back(c, &c->total_hashes, c->d_file_off.as<int64_t>() + c->nfiles, 1)))
      return rc;
    M = c->total_hashes;
    drows = c->d_hashes.as<int32_t>();
    droff = c->d_file_off.as<int64_t>();
  } else {
    if (!row_offsets || row_offsets[0] != 0) AFP_FAIL(c, AFP_ERR_INVALID, "row_offsets[0] must be 0");
    for (int f = 0; f < nfiles; ++f)
      if (row_offsets[f + 1] < row_offsets[f]) AFP_FAIL(c, AFP_ERR_INVALID, "row_offsets must be non-decreasing");
    M = row_offsets[nfiles];
    AFP_CUDA(c, c->d_st_off.reserve(sizeof(int64_t) * (size_t)(nfiles + 1)));
    AFP_CUDA(c, cudaMemcpyAsync(c->d_st_off.p, row_offsets, sizeof(int64_t) * (size_t)(nfiles + 1),
                                cudaMemcpyHostToDevice, c->stream));
    droff = c->d_st_off.as<int64_t>();
    const int rc = afp_stage(c, c->d_q, rows, 2 * (size_t)M, rows_on_host, &drows);
    if (rc) return rc;
  }
  if (M >= ((int64_t)1 << 31)) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "more than 2^31 entries in one store batch");
  for (int f = 0; f < nfiles; ++f)
    if (ids[f] < 0 || ((ids[f] + 2) << c->tab.maxtimebits) > ((int64_t)1 << 32))
      AFP_FAIL(c, AFP_ERR_INVALID, "track id does not fit in 32 - maxtimebits bits (hash_table.py:112)");
  if (M == 0) return AFP_OK;
  const int64_t nb = (int64_t)1 << c->tab.hashbits;
  AFP_CUDA(c, c->d_st_ids.reserve(sizeof(int64_t) * (size_t)nfiles));
  AFP_CUDA(c, c->d_st_eval.reserve(sizeof(uint32_t) * (size_t)M));
  AFP_CUDA(c, c->d_st_seq.reserve(sizeof(int32_t) * (size_t)M));
  AFP_CUDA(c, c->d_st_ovf.reserve(sizeof(int32_t) * (size_t)M));
  AFP_CUDA(c, c->d_st_cnt.reserve(sizeof(uint32_t) * (size_t)(2 * nb + 2)));
  AFP_CUDA(c, c->d_st_seg.reserve(sizeof(int64_t) * (size_t)(nb + 1)));
  AFP_CUDA(c, c->d_st_heavy.reserve(sizeof(int32_t) * (size_t)(M / LIGHT + 8)));
  AFP_CUDA(c, cudaMemcpyAsync(c->d_st_ids.p, ids, sizeof(int64_t) * (size_t)nfiles, cudaMemcpyHostToDevice, c->stream));
  uint32_t* cnt_new = c->d_st_cnt.as<uint32_t>();
  uint32_t* cursor = cnt_new + nb;
  int* nheavy = reinterpret_cast<int*>(cursor + nb);
  AFP_CUDA(c, cudaMemsetAsync(cnt_new, 0, sizeof(uint32_t) * (size_t)(2 * nb + 2), c->stream));
  StoreArgs a;
  a.rows = drows; a.row_off = droff; a.ids = c->d_st_ids.as<int64_t>(); a.nfiles = nfiles;
  a.hashbits = c->tab.hashbits; a.depth = c->tab.depth; a.mtb = c->tab.maxtimebits;
  a.table = c->tab.table.as<uint32_t>(); a.counts = c->tab.counts.as<int32_t>();
  a.eval = c->d_st_eval.as<uint32_t>(); a.cnt_new = cnt_new; a.seg_off = c->d_st_seg.as<int64_t>();
  a.seq = c->d_st_seq.as<int32_t>(); a.ovf_pos = c->d_st_ovf.as<int32_t>();
  a.heavy = c->d_st_heavy.as<int32_t>(); a.nheavy = nheavy;
  int h_heavy = 0;
  int rc;
  if ((rc = afp_launch(c, afp_store_count_kernel, nfiles, 256, 0, a)) ||
      (rc = afp_scan_large(c, reinterpret_cast<const int32_t*>(cnt_new), c->d_st_seg.as<int64_t>(), nb)) ||
      (rc = afp_launch(c, afp_store_scatter_kernel, (unsigned)((M + 255) / 256), 256, 0, a, M, cursor)) ||
      (rc = afp_launch(c, afp_store_place_kernel, (unsigned)((nb + 255) / 256), 256, 0, a, nb)) ||
      (rc = afp_read_back(c, &h_heavy, nheavy, 1)) ||
      (rc = afp_launch(c, afp_store_heavy_kernel, std::max(h_heavy, 0), 256, 8192 * 4, a)))
    return rc;
  // ---- overflow entries, in sequence order -------------------------------------------------
  const int64_t nblk = (M + SB - 1) / SB;
  int32_t* part = nullptr;
  int64_t* part_off = nullptr;
  int64_t novf = 0;
  if ((rc = afp_carve(c, c->d_st_part, [&](Carver& k) {
         part = k.take<int32_t>(nblk + 1);
         part_off = k.take<int64_t>(nblk + 2);
       })) ||
      (rc = afp_launch(c, afp_flag_blocksum_kernel, (unsigned)nblk, SB, 0, a.ovf_pos, M, part)) ||
      (rc = afp_scan_large(c, part, part_off, nblk)) || (rc = afp_read_back(c, &novf, part_off + nblk, 1)))
    return rc;
  if (novf > 0) {
    // sized for the whole batch at once: the overflow grows from step to step as the table fills, and
    // every regrowth would be a cudaFree + cudaMalloc in the middle of an ingest
    AFP_CUDA(c, c->d_st_obkt.reserve(sizeof(uint32_t) * (size_t)M));
    AFP_CUDA(c, c->d_st_opos.reserve(sizeof(int32_t) * (size_t)M));
    AFP_CUDA(c, c->d_st_oval.reserve(sizeof(uint32_t) * (size_t)M));
    AFP_CUDA(c, c->d_st_slot.reserve(sizeof(int32_t) * (size_t)M));
    if ((rc = afp_launch(c, afp_ovf_compact_kernel, (unsigned)nblk, SB, 0, a, M, part_off, c->d_st_obkt.as<uint32_t>(),
                         c->d_st_opos.as<int32_t>(), c->d_st_oval.as<uint32_t>())))
      return rc;
  }
  c->store_novf = novf;
  if (noverflow) *noverflow = novf;
  return AFP_OK;
}

int afp_table_fetch_overflow(afp_ctx* c, uint32_t* bucket, int32_t* count_before, uint32_t* value) {
  if (!c) return AFP_ERR_INVALID;
  AFP_CUDA(c, cudaSetDevice(c->device));
  const size_t n = (size_t)c->store_novf;
  if (!n) return afp_read_back(c);
  if (!bucket || !count_before || !value) return AFP_ERR_INVALID;
  return afp_read_back(c, bucket, c->d_st_obkt.as<uint32_t>(), n, count_before, c->d_st_opos.as<int32_t>(), n, value,
                       c->d_st_oval.as<uint32_t>(), n);
}

int afp_table_fetch_overflow_counts(afp_ctx* c, int32_t* count_before) {
  if (!c) return AFP_ERR_INVALID;
  AFP_CUDA(c, cudaSetDevice(c->device));
  const size_t n = (size_t)c->store_novf;
  if (!n) return afp_read_back(c);
  if (!count_before) return AFP_ERR_INVALID;
  return afp_read_back(c, count_before, c->d_st_opos.as<int32_t>(), n);
}

int afp_table_apply_slots(afp_ctx* c, const int32_t* slot, int64_t n) {
  if (!c || n < 0 || (n > 0 && !slot)) return AFP_ERR_INVALID;
  if (!c->tab.loaded) AFP_FAIL(c, AFP_ERR_STATE, "no table on the device");
  if (n != c->store_novf) AFP_FAIL(c, AFP_ERR_INVALID, "one slot per overflow entry of the last afp_table_store_batch");
  AFP_CUDA(c, cudaSetDevice(c->device));
  if (n == 0) return AFP_OK;
  if (n >= ((int64_t)1 << 32) - 1) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "too many overflow entries");
  const size_t cells = ((size_t)1 << c->tab.hashbits) * (size_t)c->tab.depth;
  if (c->d_st_last.cap < cells * sizeof(uint32_t)) {
    AFP_CUDA(c, c->d_st_last.reserve(cells * sizeof(uint32_t)));
    AFP_CUDA(c, cudaMemsetAsync(c->d_st_last.p, 0, cells * sizeof(uint32_t), c->stream));
  }
  AFP_CUDA(c, c->d_st_slot.reserve(sizeof(int32_t) * (size_t)n));
  AFP_CUDA(c, cudaMemcpyAsync(c->d_st_slot.p, slot, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
  const unsigned grid = (unsigned)((n + 255) / 256);
  int rc;
  if ((rc = afp_launch(c, afp_slots_mark_kernel, grid, 256, 0, c->d_st_obkt.as<uint32_t>(), c->d_st_slot.as<int32_t>(),
                       n, c->tab.depth, c->d_st_last.as<uint32_t>())) ||
      (rc = afp_launch(c, afp_slots_write_kernel, grid, 256, 0, c->d_st_obkt.as<uint32_t>(),
                       c->d_st_slot.as<int32_t>(), c->d_st_oval.as<uint32_t>(), n, c->tab.depth,
                       c->d_st_last.as<uint32_t>(), c->tab.table.as<uint32_t>())))
    return rc;
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));     // `slot` is the caller's
  c->store_novf = 0;
  return AFP_OK;
}

int afp_table_apply_patches(afp_ctx* c, const uint32_t* bucket, const int32_t* slot, const uint32_t* value, int64_t n) {
  if (!c || n < 0 || (n > 0 && (!bucket || !slot || !value))) return AFP_ERR_INVALID;
  if (!c->tab.loaded) AFP_FAIL(c, AFP_ERR_STATE, "no table on the device");
  AFP_CUDA(c, cudaSetDevice(c->device));
  if (n == 0) return AFP_OK;
  const int64_t nb = (int64_t)1 << c->tab.hashbits;
  for (int64_t i = 0; i < n; ++i)
    if ((int64_t)bucket[i] >= nb || slot[i] < 0 || slot[i] >= c->tab.depth) AFP_FAIL(c, AFP_ERR_INVALID, "patch outside the table");
  AFP_CUDA(c, c->d_st_obkt.reserve(sizeof(uint32_t) * (size_t)n));
  AFP_CUDA(c, c->d_st_opos.reserve(sizeof(int32_t) * (size_t)n));
  AFP_CUDA(c, c->d_st_oval.reserve(sizeof(uint32_t) * (size_t)n));
  AFP_CUDA(c, cudaMemcpyAsync(c->d_st_obkt.p, bucket, sizeof(uint32_t) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
  AFP_CUDA(c, cudaMemcpyAsync(c->d_st_opos.p, slot, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
  AFP_CUDA(c, cudaMemcpyAsync(c->d_st_oval.p, value, sizeof(uint32_t) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
  const int rc = afp_launch(c, afp_patch_kernel, (unsigned)((n + 255) / 256), 256, 0, c->tab.table.as<uint32_t>(),
                            c->tab.depth, c->d_st_obkt.as<uint32_t>(), c->d_st_opos.as<int32_t>(),
                            c->d_st_oval.as<uint32_t>(), n);
  if (rc) return rc;
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  return AFP_OK;
}

int afp_table_download(afp_ctx* c, uint32_t* table, int32_t* counts) {
  if (!c || !table || !counts) return AFP_ERR_INVALID;
  if (!c->tab.loaded) AFP_FAIL(c, AFP_ERR_STATE, "no table on the device");
  AFP_CUDA(c, cudaSetDevice(c->device));
  const size_t nb = (size_t)1 << c->tab.hashbits;
  return afp_read_back(c, table, c->tab.table.as<uint32_t>(), nb * (size_t)c->tab.depth, counts,
                       c->tab.counts.as<int32_t>(), nb);
}

// ---- CPython's random.randint(0, count) replayed in C (host bookkeeping, not the hot path) ----
// state = random.getstate()[1]: 624 words of MT19937 state + the position (625 uint32).
// random.randint(a, b) -> randrange(a, b + 1) -> a + _randbelow(b - a + 1);
// _randbelow_with_getrandbits(n): k = n.bit_length(); r = getrandbits(k); while r >= n: r = getrandbits(k)
// getrandbits(k <= 32) = genrand_uint32() >> (32 - k)        (Lib/random.py, Modules/_randommodule.c)
static inline uint32_t mt_next(uint32_t* mt, uint32_t* pos) {
  constexpr int N = 624, Mm = 397;
  if (*pos >= (uint32_t)N) {
    int kk;
    for (kk = 0; kk < N - Mm; ++kk) {
      const uint32_t y = (mt[kk] & 0x80000000u) | (mt[kk + 1] & 0x7fffffffu);
      mt[kk] = mt[kk + Mm] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    for (; kk < N - 1; ++kk) {
      const uint32_t y = (mt[kk] & 0x80000000u) | (mt[kk + 1] & 0x7fffffffu);
      mt[kk] = mt[kk + (Mm - N)] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    const uint32_t y = (mt[N - 1] & 0x80000000u) | (mt[0] & 0x7fffffffu);
    mt[N - 1] = mt[Mm - 1] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    *pos = 0;
  }
  uint32_t y = mt[(*pos)++];
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= y >> 18;
  return y;
}

int afp_mt_randint_replay(uint32_t* state625, const int32_t* count_before, int64_t n, int32_t* slot_out) {
  if (!state625 || n < 0 || (n > 0 && (!count_before || !slot_out))) return AFP_ERR_INVALID;
  uint32_t pos = state625[624];
  if (pos > 624u) return AFP_ERR_INVALID;
  for (int64_t i = 0; i < n; ++i) {
    if (count_before[i] < 0) return AFP_ERR_INVALID;
    const uint32_t width = (uint32_t)count_before[i] + 1u;     // randint(0, count): count + 1 values
    int k = 32 - __builtin_clz(width);                          // width.bit_length(), width >= 1
    uint32_t r = mt_next(state625, &pos) >> (32 - k);
    while (r >= width) r = mt_next(state625, &pos) >> (32 - k);
    slot_out[i] = (int32_t)r;
  }
  state625[624] = pos;
  return AFP_OK;
}

}  // extern "C"

// int32[n] -> exclusive int64[n+1], any n (block sums, scan of the sums, per-block scan with carry)
namespace {
__global__ void __launch_bounds__(SB) afp_blocksum_kernel(const int32_t* in, int64_t n, int64_t* part) {
  __shared__ long long s[SB / 32];
  const int64_t i = (int64_t)blockIdx.x * SB + threadIdx.x;
  long long v = i < n ? in[i] : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long t = 0;
    for (int w = 0; w < SB / 32; ++w) t += s[w];
    part[blockIdx.x] = t;
  }
}
// in-place exclusive scan of up to a few thousand partial sums by one CTA; total at part[nblk]
__global__ void __launch_bounds__(SB) afp_partscan_kernel(int64_t* part, int64_t nblk) {
  __shared__ long long s[SB];
  __shared__ long long run;
  if (threadIdx.x == 0) run = 0;
  __syncthreads();
  for (int64_t i0 = 0; i0 < nblk; i0 += SB) {
    const int64_t i = i0 + threadIdx.x;
    const long long c = i < nblk ? part[i] : 0;
    s[threadIdx.x] = c;
    __syncthreads();
    for (int o = 1; o < SB; o <<= 1) {
      const long long v = threadIdx.x >= o ? s[threadIdx.x - o] : 0;
      __syncthreads();
      s[threadIdx.x] += v;
      __syncthreads();
    }
    if (i < nblk) part[i] = s[threadIdx.x] - c + run;
    __syncthreads();
    if (threadIdx.x == SB - 1) run += s[SB - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[nblk] = run;
}
__global__ void __launch_bounds__(SB) afp_blockscan_kernel(const int32_t* in, int64_t n, const int64_t* part, int64_t* out) {
  __shared__ long long s[SB / 32];
  const int64_t i = (int64_t)blockIdx.x * SB + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long c = i < n ? in[i] : 0;
  long long v = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  if (lane == 31) s[warp] = v;
  __syncthreads();
  if (warp == 0) {
    long long w = s[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long t = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += t;
    }
    s[lane] = w;
  }
  __syncthreads();
  if (i < n) out[i] = part[blockIdx.x] + (warp ? s[warp - 1] : 0) + v - c;
  if (i == n - 1) out[n] = part[blockIdx.x] + (warp ? s[warp - 1] : 0) + v;
}
}  // namespace

int afp_scan_large(afp_ctx* c, const int32_t* in, int64_t* out, int64_t n) {
  if (n <= 0) {
    AFP_CUDA(c, cudaMemsetAsync(out, 0, sizeof(int64_t), c->stream));
    return AFP_OK;
  }
  const int64_t nblk = (n + SB - 1) / SB;
  AFP_CUDA(c, c->d_st_scan.reserve(sizeof(int64_t) * (size_t)(nblk + 2)));
  int64_t* part = c->d_st_scan.as<int64_t>();
  int rc;
  if ((rc = afp_launch(c, afp_blocksum_kernel, (unsigned)nblk, SB, 0, in, n, part)) ||
      (rc = afp_launch(c, afp_partscan_kernel, 1, SB, 0, part, nblk)))
    return rc;
  return afp_launch(c, afp_blockscan_kernel, (unsigned)nblk, SB, 0, in, n, part, out);
}
