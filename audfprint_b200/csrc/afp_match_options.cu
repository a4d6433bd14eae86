// The matcher's second-wave options on the device: exact distinct-hash counts (exact_count,
// _exact_match_counts / _unique_match_hashes, audfprint_match.py:149-171 and :196-239) and
// query time ranges (find_time_range, _calculate_time_ranges, :173-194), for a whole batch.
//
// afp_match_options_batch ranks the queries with afp_match_batch in publish mode (fast, general
// and long-query kernels alike), then finishes on the device without materialising the hits:
//   1. slots: every (query, rank < depth) whose raw count reaches max(threshcount, 1) is routed;
//      its segment is raw entries long (a scan lays the segments out), and the query's routed ids
//      are sorted by id (CUB segmented sort) for the lookup of step 2;
//   2. probe: one grid-wide pass over all query rows of the batch, one warp per row; every hit of
//      a routed id (binary search in its query's sorted ids) goes to that candidate's segment as
//      (dtime, qtime, hash).  The same pass takes each query's largest qtime over ALL its hits;
//   3. each segment is sorted by dtime (CUB segmented sort): equal dtimes form the bins of the
//      reference's dense histogram, so locmax / find_modes (:51-90) read neighbouring runs;
//   4. modes: exact_count - every run that is a local maximum and reaches threshcount, in
//      (query, rank, dtime) order; find_time_range alone - the approximate rows of rank < depth;
//   5. supports: the entries within +-window of each mode, copied out as packed keys
//      qtime + (hash << timebits) and/or qtimes, each support sorted (CUB segmented sort): the
//      distinct count is the number of key runs, the quantiles are two indexed reads;
//   6. rows: flagged (count >= threshcount), scanned and written in mode order.
// timebits = max(1, ceil(log(qmax)/log(2))) is evaluated with the caller's 32 breakpoints of that
// expression, so that its power-of-two shortfall (and the key collisions that follow) are the
// reference's.  Memory: the routed candidates' hits and their supports - an entry lies in at most
// window + 1 exact-count supports (modes are at least two bins apart) and in at most 2 approximate
// ones - plus O(nqueries * search_depth); nothing is sized by rows x depth.  Every result is read
// from sorted data, so nothing depends on the order of the probe's atomics.
//
// A shard of an id-range sharded table runs the same finish in two calls around the caller's
// all-reduce (MAX) of each query's largest qtime (afp_match_options_shard_rank / _finish): every
// published candidate is finished (the merge keeps global ranks < D), the key width comes from the
// reduced maximum, and a failed quantile read is recorded per query for the merge (afp_shard.cu).
#include <math.h>
#include <algorithm>
#include <cub/cub.cuh>
#include "afp_internal.cuh"

namespace {

constexpr int OT = 256;

struct Breaks {
  long long v[32];     // v[k-1] = smallest qmax whose ceil(log(qmax)/log(2)) >= k
};

__device__ __forceinline__ int timebits_of(const Breaks& b, int qmax) {
  int t = 0;
#pragma unroll
  for (int k = 0; k < 32; ++k) t += (long long)qmax >= b.v[k] ? 1 : 0;
  return max(1, t);
}

// first index in [lo, hi) whose value is >= x (strict = false) or > x (strict = true)
template <class T>
__device__ __forceinline__ int64_t bound(const T* v, int64_t lo, int64_t hi, long long x, bool strict) {
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    const long long y = (long long)v[mid];
    if (strict ? y <= x : y < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// candidates finished per query: a whole table reaches rank min(n_above, search_depth) (:139-146);
// a shard of an id-range sharded table finishes every candidate it publishes, because one of its
// ids can be inside the global top-D while at or past the shard's own n_above (the merge drops
// the rows of global rank >= D)
__device__ __forceinline__ int depth_of(const int32_t* cnt, int qi, int sd, int shard) {
  return max(0, min(shard ? sd : min(cnt[2 * qi + 1], sd), cnt[2 * qi]));
}

// 1. per (query, rank) slot: segment length, lookup key (id, or ~0 when not routed) and rank
__global__ void opt_slots_kernel(const double* cand, const int32_t* cnt, int nq, int sd, int thresh, int shard,
                                 int64_t* seglen, uint32_t* lkey, int32_t* lval, int32_t* loff, int* qmax) {
  const int64_t n = (int64_t)nq * sd;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (int64_t)gridDim.x * blockDim.x) {
    if (i <= nq) loff[i] = (int32_t)(i * sd);
    if (i < nq) qmax[i] = 0;
    if (i == n) { seglen[n] = 0; continue; }
    const int qi = (int)(i / sd), j = (int)(i % sd);
    bool routed = false;
    int raw = 0;
    uint32_t id = 0xffffffffu;
    if (j < depth_of(cnt, qi, sd, shard)) {
      raw = (int)cand[3 * i + 1];
      routed = raw >= max(thresh, 1);          // find_modes keeps bins >= threshcount (:78-90)
      if (routed) id = (uint32_t)cand[3 * i];
    }
    seglen[i] = routed ? raw : 0;
    lkey[i] = id;
    lval[i] = j;
  }
}

// 2. one warp per query row: route the hits of routed ids to their segments
__global__ void __launch_bounds__(OT) opt_probe_kernel(const int32_t* q, int64_t nrows, const int64_t* qoff, int nq,
                                                       const uint32_t* table, const int32_t* counts, int hashbits,
                                                       int depth, int mtb, int64_t nids, int sd, const uint32_t* lkey,
                                                       const int32_t* lval, const int64_t* segoff, unsigned* cur,
                                                       int32_t* dt, unsigned long long* pay, int32_t* hseg, int* qmax,
                                                       int* err) {
  const int lane = threadIdx.x & 31;
  const uint32_t hmask = (1u << hashbits) - 1u, tmask = (1u << mtb) - 1u;
  const int64_t nwarps = (int64_t)gridDim.x * (OT / 32);
  for (int64_t r = (int64_t)blockIdx.x * (OT / 32) + (threadIdx.x >> 5); r < nrows; r += nwarps) {
    const int qi = (int)bound(qoff, 0, nq + 1, r, true) - 1;     // qoff[qi] <= r < qoff[qi + 1]
    const int qt = q[2 * r];
    const uint32_t b = (uint32_t)q[2 * r + 1] & hmask;
    const int nb = min(depth, counts[b]);
    if (nb > 0 && lane == 0) atomicMax(&qmax[qi], qt);          // timebits: over all hits of the query
    const uint32_t* L = lkey + (size_t)qi * sd;
    const uint32_t* row = table + (size_t)b * depth;
    for (int s = lane; s < nb; s += 32) {
      const uint32_t v = row[s];
      const uint32_t id = (v >> mtb) - 1u;
      if (id >= (uint32_t)nids) continue;
      const int k = (int)bound(L, 0, sd, id, false);
      if (k >= sd || L[k] != id) continue;
      const int64_t slot = (int64_t)qi * sd + lval[(size_t)qi * sd + k];
      const int64_t p = segoff[slot] + atomicAdd(&cur[slot], 1u);
      if (p >= segoff[slot + 1]) { atomicExch(err, 1); continue; }
      dt[p] = (int32_t)(v & tmask) - qt;
      pay[p] = ((unsigned long long)b << 32) | (uint32_t)qt;
      hseg[p] = (int32_t)slot;
    }
  }
}

// every segment must have been filled to its raw count exactly
__global__ void opt_fill_check_kernel(const int64_t* seglen, const unsigned* cur, int64_t n, int* err) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if ((int64_t)cur[i] != seglen[i]) atomicExch(err, 1);
}

// 4a. exact_count: flag the first entry of every dtime run that is a mode - locmax of the dense
// histogram (>= the previous bin, > the next; no test beyond either end) and >= threshcount
__global__ void opt_modes_kernel(const int32_t* dt, const int32_t* hseg, const int64_t* segoff, int64_t h, int thresh,
                                 int32_t* flag) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= h; i += (int64_t)gridDim.x * blockDim.x) {
    if (i == h) { flag[h] = 0; continue; }
    const int s = hseg[i];
    const int64_t s0 = segoff[s], s1 = segoff[s + 1];
    const long long d = dt[i];
    if (i > s0 && dt[i - 1] == d) { flag[i] = 0; continue; }
    const int64_t end = bound(dt, i, s1, d, true);
    const int64_t c = end - i;
    const int64_t pc = (i > s0 && dt[i - 1] == d - 1) ? i - bound(dt, s0, i, d - 1, false) : 0;
    const int64_t nc = (end < s1 && dt[end] == d + 1) ? bound(dt, end, s1, d + 1, true) - end : 0;
    flag[i] = (c >= pc && nc < c && c >= thresh) ? 1 : 0;
  }
}

// 4b. find_time_range alone: flag the approximate rows of rank < depth
__global__ void opt_rowflags_kernel(const int32_t* rows, int64_t nr, const int64_t* roff, int nq, const int32_t* cnt,
                                    int sd, int shard, int32_t* flag) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= nr; r += (int64_t)gridDim.x * blockDim.x) {
    if (r == nr) { flag[nr] = 0; continue; }
    const int qi = (int)bound(roff, 0, nq + 1, r, true) - 1;
    flag[r] = rows[7 * r + 4] < depth_of(cnt, qi, sd, shard) ? 1 : 0;
  }
}

// order-preserving compaction: out[pos[i]] = i for every flagged i
__global__ void opt_scatter_kernel(const int32_t* flag, const int32_t* pos, int64_t n, int32_t* out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (flag[i]) out[pos[i]] = (int32_t)i;
}

// 5a. every mode: its slot, dtime and support [lo, lo + len) in its segment
__global__ void opt_support_kernel(const int32_t* midx, int nm, int exact, const int32_t* dt, const int32_t* hseg,
                                   const int64_t* segoff, const int32_t* rows, const int64_t* roff, int nq, int sd,
                                   int window, int32_t* mslot, int32_t* mdt, int64_t* mlo, int64_t* slen) {
  for (int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; m <= nm; m += (int64_t)gridDim.x * blockDim.x) {
    if (m == nm) { slen[nm] = 0; continue; }
    const int src = midx[m];
    int s, d;
    if (exact) {
      s = hseg[src];
      d = dt[src];
    } else {
      const int qi = (int)bound(roff, 0, nq + 1, src, true) - 1;
      s = qi * sd + rows[7 * (int64_t)src + 4];
      d = rows[7 * (int64_t)src + 2];
    }
    const int64_t s0 = segoff[s], s1 = segoff[s + 1];
    const int64_t lo = bound(dt, s0, s1, (long long)d - window, false);
    const int64_t hi = bound(dt, lo, s1, (long long)d + window, true);
    mslot[m] = s;
    mdt[m] = d;
    mlo[m] = lo;
    slen[m] = hi - lo;
  }
}

// 5b. copy every support out: packed keys (exact_count) and qtimes (find_time_range)
__global__ void opt_gather_kernel(const int64_t* soff, int nm, const int64_t* mlo, const int32_t* mslot, int sd,
                                  const unsigned long long* pay, const int* qmax, Breaks br, unsigned long long* pk,
                                  int32_t* tq) {
  const int64_t total = soff[nm];
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
    const int m = (int)bound(soff, 0, nm + 1, p, true) - 1;
    const unsigned long long v = pay[mlo[m] + (p - soff[m])];
    const uint32_t qt = (uint32_t)v;
    if (pk) pk[p] = (unsigned long long)qt + ((v >> 32) << timebits_of(br, qmax[mslot[m] / sd]));
    if (tq) tq[p] = (int32_t)qt;
  }
}

// Python's t[i] index: negative wraps once, anything else outside [0, n) is an IndexError
__device__ __forceinline__ bool py_index(double x, int64_t n, int64_t& i) {
  const double t = trunc(x);
  if (!(t >= -(double)n && t < (double)n)) return false;
  i = (int64_t)t;
  if (i < 0) i += n;
  return true;
}

// 5c. one warp per mode: distinct keys of its sorted support, the two quantile reads, the row flag.
// A failed quantile read is an error of the call (err), or on a shard (qfail != nullptr) the
// candidate's local rank, kept per query (the smallest) for the merge to judge
__global__ void __launch_bounds__(OT) opt_stats_kernel(const int64_t* soff, int nm, const unsigned long long* pk,
                                                       const int32_t* tq, int thresh, double quant, const int32_t* mslot,
                                                       int sd, int32_t* mcnt, int32_t* mtlo, int32_t* mthi,
                                                       int32_t* keep, int* err, int32_t* qfail) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t)gridDim.x * (OT / 32);
  for (int64_t m = (int64_t)blockIdx.x * (OT / 32) + (threadIdx.x >> 5); m <= nm; m += nwarps) {
    if (m == nm) { if (lane == 0) keep[nm] = 0; continue; }
    const int64_t a = soff[m], n = soff[m + 1] - a;
    bool k = true;
    if (pk) {
      int c = 0;
      for (int64_t p = a + lane; p < a + n; p += 32) c += (p == a || pk[p] != pk[p - 1]) ? 1 : 0;
      c = __reduce_add_sync(0xffffffffu, c);
      k = c >= thresh;
      if (lane == 0) mcnt[m] = c;
    }
    if (lane == 0) {
      keep[m] = k ? 1 : 0;
      if (tq && k) {
        int64_t ilo, ihi;
        if (py_index((double)n * quant, n, ilo) && py_index(trunc((double)n * (1.0 - quant)) - 1.0, n, ihi)) {
          mtlo[m] = tq[a + ilo];
          mthi[m] = tq[a + ihi];
        } else if (qfail) {
          mtlo[m] = mthi[m] = 0;
          atomicMin(&qfail[mslot[m] / sd], mslot[m] % sd);
        } else {
          atomicExch(err, 1);
        }
      }
    }
  }
}

// 6. the rows, in mode order; per-query row counts
__global__ void opt_rows_kernel(int nm, const int32_t* keep, const int32_t* kpos, const int32_t* midx,
                                const int32_t* mslot, const int32_t* mdt, const int32_t* mcnt, const int32_t* mtlo,
                                const int32_t* mthi, int exact, int trange, const double* cand, int sd,
                                const int32_t* approx, int32_t* out, unsigned long long* qcnt) {
  for (int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; m < nm; m += (int64_t)gridDim.x * blockDim.x) {
    if (!keep[m]) continue;
    const int s = mslot[m];
    int32_t* o = out + 7 * (int64_t)kpos[m];
    if (exact) {
      o[0] = (int32_t)cand[3 * (int64_t)s];
      o[1] = mcnt[m];
      o[2] = mdt[m];
      o[3] = (int32_t)cand[3 * (int64_t)s + 1];
      o[4] = s % sd;
    } else {
      for (int e = 0; e < 5; ++e) o[e] = approx[7 * (int64_t)midx[m] + e];
    }
    o[5] = trange ? mtlo[m] : 0;
    o[6] = trange ? mthi[m] : 0;
    atomicAdd(&qcnt[s / sd], 1ull);
  }
}

unsigned grid_for(int64_t n, int threads) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + threads - 1) / threads, 132 * 32));
}

// The finish on the ranking afp_match_batch left in the context (publish mode).  On a shard
// (qmax_shard != nullptr): every published candidate is finished, the key width comes from the
// caller's per-query largest qtime over ALL shards, and quantile failures go to qfail.
int finish_options(afp_ctx* c, const int32_t* dq, int nq, int64_t nrows, int64_t napprox, const afp_matcher_params* p,
                   int exact, int trange, double quant, const Breaks& br, const int* qmax_shard, int32_t* qfail,
                   int64_t* total_out) {
  cudaStream_t st = c->stream;
  const int shard = qmax_shard ? 1 : 0;
  const int sd = p->search_depth, thresh = p->threshcount, window = p->window;
  const int64_t nslot = (int64_t)nq * sd;
  if (nslot >= ((int64_t)1 << 31)) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "nqueries * search_depth >= 2^31");
  const double* cand = c->d_mcand.as<double>();
  const int32_t* cnt = c->d_mcand_cnt.as<int32_t>();
  int rc;
  // ---- 1. slots, segments, sorted lookup ids
  int64_t *seglen, *segoff;
  uint32_t *lkey, *lkey2;
  int32_t *lval, *lval2, *loff;
  unsigned* cur;
  int *qmax, *err;
  unsigned long long* qcnt;
  if ((rc = afp_carve(c, c->d_op_slot, [&](Carver& k) {
         seglen = k.take<int64_t>(nslot + 1);
         segoff = k.take<int64_t>(nslot + 1);
         lkey = k.take<uint32_t>(nslot);
         lkey2 = k.take<uint32_t>(nslot);
         lval = k.take<int32_t>(nslot);
         lval2 = k.take<int32_t>(nslot);
         loff = k.take<int32_t>(nq + 1);
         cur = k.take<unsigned>(nslot);
         qmax = k.take<int>(nq);
         err = k.take<int>(4);
         qcnt = k.take<unsigned long long>(nq + 1);
       })))
    return rc;
  AFP_CUDA(c, cudaMemsetAsync(cur, 0, sizeof(unsigned) * (size_t)std::max<int64_t>(nslot, 1), st));
  AFP_CUDA(c, cudaMemsetAsync(err, 0, sizeof(int) * 4, st));
  AFP_CUDA(c, cudaMemsetAsync(qcnt, 0, sizeof(unsigned long long) * (size_t)(nq + 1), st));
  if ((rc = afp_launch(c, opt_slots_kernel, grid_for(nslot + 1, OT), OT, 0, cand, cnt, nq, sd, thresh, shard, seglen,
                       lkey, lval, loff, qmax)))
    return rc;
  if ((rc = cub_call(c, [&](void* t, size_t& b) {
         return cub::DeviceScan::ExclusiveSum(t, b, seglen, segoff, (int)(nslot + 1), st);
       })))
    return rc;
  if ((rc = cub_call(c, [&](void* t, size_t& b) {
         return cub::DeviceSegmentedRadixSort::SortPairs(t, b, lkey, lkey2, lval, lval2, (int)nslot, nq, loff, loff + 1,
                                                         0, 32, st);
       })))
    return rc;
  int64_t nh = 0;
  if ((rc = afp_read_back(c, &nh, segoff + nslot, 1))) return rc;
  if (nh >= ((int64_t)1 << 31)) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "the candidates' hits of one call reach 2^31");
  // ---- 2. probe: the routed candidates' hits into their segments
  int32_t *dt, *dt2, *hseg, *flag, *pos;
  unsigned long long *pay, *pay2;
  if ((rc = afp_carve(c, c->d_op_hit, [&](Carver& k) {
         dt = k.take<int32_t>(nh);
         dt2 = k.take<int32_t>(nh);
         pay = k.take<unsigned long long>(nh);
         pay2 = k.take<unsigned long long>(nh);
         hseg = k.take<int32_t>(nh);
         flag = k.take<int32_t>(nh + 1);
         pos = k.take<int32_t>(nh + 1);
       })))
    return rc;
  if (nrows > 0 &&
      (rc = afp_launch(c, opt_probe_kernel, grid_for(nrows, OT / 32), OT, 0, dq, nrows, c->d_qoff.as<int64_t>(), nq,
                       c->tab.table.as<uint32_t>(), c->tab.counts.as<int32_t>(), c->tab.hashbits, c->tab.depth,
                       c->tab.maxtimebits, std::max<int64_t>(c->tab.nids, 1), sd, lkey2, lval2, segoff, cur, dt, pay,
                       hseg, qmax, err)))
    return rc;
  if (nslot > 0 && (rc = afp_launch(c, opt_fill_check_kernel, grid_for(nslot, OT), OT, 0, seglen, cur, nslot, err)))
    return rc;
  // ---- 3. every segment by dtime
  if (nh > 0 && (rc = cub_call(c, [&](void* t, size_t& b) {
                   return cub::DeviceSegmentedSort::SortPairs(t, b, dt, dt2, pay, pay2, (int)nh, (int)nslot, segoff,
                                                              segoff + 1, st);
                 })))
    return rc;
  // ---- 4. modes (as positions of their first entry, or as approximate row numbers)
  const int32_t* approx = c->d_mrows_packed.as<int32_t>();
  const int64_t* roff = c->d_mrow_off.as<int64_t>();
  const int64_t nsrc = exact ? nh : napprox;
  if (!exact) {
    if ((rc = afp_carve(c, c->d_op_mode, [&](Carver& k) {
           flag = k.take<int32_t>(nsrc + 1);
           pos = k.take<int32_t>(nsrc + 1);
         })))
      return rc;
    rc = afp_launch(c, opt_rowflags_kernel, grid_for(nsrc + 1, OT), OT, 0, approx, nsrc, roff, nq, cnt, sd, shard, flag);
  } else {
    rc = afp_launch(c, opt_modes_kernel, grid_for(nsrc + 1, OT), OT, 0, dt2, hseg, segoff, nsrc, thresh, flag);
  }
  if (rc) return rc;
  if ((rc = cub_call(c, [&](void* t, size_t& b) {
         return cub::DeviceScan::ExclusiveSum(t, b, flag, pos, (int)(nsrc + 1), st);
       })))
    return rc;
  int h_m[2] = {0, 0};
  if ((rc = afp_read_back(c, &h_m[0], pos + nsrc, 1, &h_m[1], err, 1))) return rc;
  if (h_m[1]) AFP_FAIL(c, AFP_ERR_STATE, "a candidate's hits differ from its raw count (table changed during the call?)");
  const int nm = h_m[0];
  // ---- 5. supports
  int32_t *midx, *mslot, *mdt, *mcnt, *mtlo, *mthi, *keep, *kpos;
  int64_t *mlo, *slen, *soff;
  if ((rc = afp_carve(c, c->d_op_sup, [&](Carver& k) {
         midx = k.take<int32_t>(nm);
         mslot = k.take<int32_t>(nm);
         mdt = k.take<int32_t>(nm);
         mcnt = k.take<int32_t>(nm);
         mtlo = k.take<int32_t>(nm);
         mthi = k.take<int32_t>(nm);
         keep = k.take<int32_t>(nm + 1);
         kpos = k.take<int32_t>(nm + 1);
         mlo = k.take<int64_t>(nm);
         slen = k.take<int64_t>(nm + 1);
         soff = k.take<int64_t>(nm + 1);
       })))
    return rc;
  if (nsrc > 0 && (rc = afp_launch(c, opt_scatter_kernel, grid_for(nsrc, OT), OT, 0, flag, pos, nsrc, midx))) return rc;
  if ((rc = afp_launch(c, opt_support_kernel, grid_for(nm + 1, OT), OT, 0, midx, nm, exact, dt2, hseg, segoff, approx,
                       roff, nq, sd, window, mslot, mdt, mlo, slen)))
    return rc;
  if ((rc = cub_call(c, [&](void* t, size_t& b) {
         return cub::DeviceScan::ExclusiveSum(t, b, slen, soff, nm + 1, st);
       })))
    return rc;
  int64_t ns = 0;
  if ((rc = afp_read_back(c, &ns, soff + nm, 1))) return rc;
  if (ns >= ((int64_t)1 << 31)) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "the mode supports of one call reach 2^31 entries");
  unsigned long long *pk = nullptr, *pk2 = nullptr;
  int32_t *tq = nullptr, *tq2 = nullptr;
  if (exact && (rc = afp_carve(c, c->d_op_key, [&](Carver& k) {
                  pk = k.take<unsigned long long>(ns);
                  pk2 = k.take<unsigned long long>(ns);
                })))
    return rc;
  if (trange && (rc = afp_carve(c, c->d_op_tq, [&](Carver& k) {
                   tq = k.take<int32_t>(ns);
                   tq2 = k.take<int32_t>(ns);
                 })))
    return rc;
  if (ns > 0) {
    if ((rc = afp_launch(c, opt_gather_kernel, grid_for(ns, OT), OT, 0, soff, nm, mlo, mslot, sd, pay2,
                         shard ? qmax_shard : qmax, br, pk, tq)))
      return rc;
    if (exact && (rc = cub_call(c, [&](void* t, size_t& b) {
                    return cub::DeviceSegmentedSort::SortKeys(t, b, pk, pk2, (int)ns, nm, soff, soff + 1, st);
                  })))
      return rc;
    if (trange && (rc = cub_call(c, [&](void* t, size_t& b) {
                     return cub::DeviceSegmentedSort::SortKeys(t, b, tq, tq2, (int)ns, nm, soff, soff + 1, st);
                   })))
      return rc;
  }
  // ---- 6. counts, quantiles, rows
  if ((rc = afp_launch(c, opt_stats_kernel, grid_for(nm + 1, OT / 32), OT, 0, soff, nm, pk2, tq2, thresh, quant, mslot,
                       sd, mcnt, mtlo, mthi, keep, err + 1, qfail)))
    return rc;
  if ((rc = cub_call(c, [&](void* t, size_t& b) {
         return cub::DeviceScan::ExclusiveSum(t, b, keep, kpos, nm + 1, st);
       })))
    return rc;
  int h_r[2] = {0, 0};
  if ((rc = afp_read_back(c, &h_r[0], kpos + nm, 1, &h_r[1], err + 1, 1))) return rc;
  if (h_r[1]) AFP_FAIL(c, AFP_ERR_INDEX, "time_quantile index outside a support (IndexError)");
  const int nr = h_r[0];
  AFP_CUDA(c, c->d_op_rows.reserve(sizeof(int32_t) * 7 * (size_t)(nr + 1)));
  if (nm > 0 &&
      (rc = afp_launch(c, opt_rows_kernel, grid_for(nm, OT), OT, 0, nm, keep, kpos, midx, mslot, mdt, mcnt, mtlo, mthi,
                       exact, trange, cand, sd, approx, c->d_op_rows.as<int32_t>(), qcnt)))
    return rc;
  static_assert(sizeof(unsigned long long) == sizeof(int64_t), "row counts scan in place of int64 offsets");
  if ((rc = cub_call(c, [&](void* t, size_t& b) {
         return cub::DeviceScan::ExclusiveSum(t, b, reinterpret_cast<int64_t*>(qcnt), c->d_mrow_off.as<int64_t>(),
                                              nq + 1, st);
       })))
    return rc;
  std::swap(c->d_mrows_packed, c->d_op_rows);      // afp_fetch_match_rows returns the finished rows
  AFP_CUDA(c, cudaStreamSynchronize(st));
  *total_out = nr;
  return AFP_OK;
}

// a shard's largest query time over the query rows whose bucket is non-empty on it - the rows the
// probe's atomicMax reads (step 2), so that the maximum over the shards is the whole table's
__global__ void opt_shard_qmax_kernel(const int32_t* q, int64_t nrows, const int64_t* qoff, int nq,
                                      const int32_t* counts, int hashbits, int depth, int* qmax) {
  const uint32_t hmask = (1u << hashbits) - 1u;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
    if (min(depth, counts[(uint32_t)q[2 * r + 1] & hmask]) <= 0) continue;
    const int qi = (int)bound(qoff, 0, nq + 1, r, true) - 1;
    atomicMax(&qmax[qi], q[2 * r]);
  }
}

// argument checks and the ranking (publish mode) shared by the whole-table and the shard form
int rank_options(afp_ctx* c, const int32_t* q_rows, int q_on_host, int32_t nqueries, const int64_t* q_offsets,
                 const afp_matcher_params* p, int32_t exact_count, int32_t find_time_range, double time_quantile,
                 const int64_t* timebits_breaks, Breaks& br, int64_t* ranked, const int32_t** dq) {
  if (!c || !p || !timebits_breaks) return AFP_ERR_INVALID;
  if ((exact_count != 0 && exact_count != 1) || (find_time_range != 0 && find_time_range != 1) ||
      !(exact_count || find_time_range))
    AFP_FAIL(c, AFP_ERR_INVALID, "exact_count and find_time_range are 0 or 1, and one of them is 1");
  if (!isfinite(time_quantile)) AFP_FAIL(c, AFP_ERR_INVALID, "time_quantile must be finite");
  if (p->window < 0 || p->window > 4096 || p->threshcount < 0 || p->search_depth < 0 || p->max_alignments_per_id < 0)
    AFP_FAIL(c, AFP_ERR_INVALID, "bad matcher parameters");
  for (int k = 0; k < 32; ++k) {
    br.v[k] = timebits_breaks[k];
    if (br.v[k] < 1 || (k > 0 && br.v[k] < br.v[k - 1]))
      AFP_FAIL(c, AFP_ERR_INVALID, "timebits breakpoints must be positive and non-decreasing");
  }
  // ranking in publish mode.  exact_count needs no approximate rows: at most one per candidate
  // (max_alignments_per_id 0) and room for all of them, so that the ranking never overflows.
  afp_matcher_params rp = *p;
  rp.publish_candidates = 1;
  if (exact_count) {
    rp.max_alignments_per_id = 0;
    rp.row_capacity = std::max(p->row_capacity > 0 ? p->row_capacity : 256, p->search_depth);
  }
  *ranked = 0;
  int rc = afp_match_batch(c, q_rows, q_on_host, nqueries, q_offsets, &rp, ranked);
  if (rc) return rc;
  const int64_t nrows = nqueries ? q_offsets[nqueries] : 0;
  *dq = (q_on_host && nrows > 0) ? c->d_q.as<int32_t>() : q_rows;
  return AFP_OK;
}

}  // namespace

extern "C" int afp_match_options_batch(afp_ctx* c, const int32_t* q_rows, int q_on_host, int32_t nqueries,
                                       const int64_t* q_offsets, const afp_matcher_params* p, int32_t exact_count,
                                       int32_t find_time_range, double time_quantile, const int64_t* timebits_breaks,
                                       int64_t* total_rows) {
  Breaks br;
  int64_t ranked = 0;
  const int32_t* dq = nullptr;
  int rc = rank_options(c, q_rows, q_on_host, nqueries, q_offsets, p, exact_count, find_time_range, time_quantile,
                        timebits_breaks, br, &ranked, &dq);
  if (rc) return rc;
  const int64_t nrows = nqueries ? q_offsets[nqueries] : 0;
  int64_t total = 0;
  c->match_total_rows = -1;                 // the approximate rows are not this call's result
  if (nqueries > 0 && p->search_depth > 0) {
    if ((rc = finish_options(c, dq, nqueries, nrows, ranked, p, exact_count, find_time_range, time_quantile, br,
                             nullptr, nullptr, &total)))
      return rc;
  } else if (nqueries > 0) {
    AFP_CUDA(c, cudaMemsetAsync(c->d_mrow_off.p, 0, sizeof(int64_t) * (size_t)(nqueries + 1), c->stream));
    AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  }
  c->match_total_rows = total;
  if (total_rows) *total_rows = total;
  return AFP_OK;
}

extern "C" int afp_match_options_shard_rank(afp_ctx* c, const int32_t* q_rows, int q_on_host, int32_t nqueries,
                                            const int64_t* q_offsets, const afp_matcher_params* p,
                                            int32_t exact_count, int32_t find_time_range, double time_quantile,
                                            const int64_t* timebits_breaks, int32_t* qmax_dev, int64_t* ranked_rows) {
  if (c) c->sopt.pending = c->sopt.finished = false;
  if (c && nqueries > 0 && !qmax_dev) return AFP_ERR_INVALID;
  Breaks br;
  int64_t ranked = 0;
  const int32_t* dq = nullptr;
  int rc = rank_options(c, q_rows, q_on_host, nqueries, q_offsets, p, exact_count, find_time_range, time_quantile,
                        timebits_breaks, br, &ranked, &dq);
  if (rc) return rc;
  const int64_t nrows = nqueries ? q_offsets[nqueries] : 0;
  if (nqueries > 0) {
    AFP_CUDA(c, cudaMemsetAsync(qmax_dev, 0, sizeof(int32_t) * (size_t)nqueries, c->stream));
    if (nrows > 0 &&
        (rc = afp_launch(c, opt_shard_qmax_kernel, grid_for(nrows, OT), OT, 0, dq, nrows, c->d_qoff.as<int64_t>(),
                         nqueries, c->tab.counts.as<int32_t>(), c->tab.hashbits, c->tab.depth, qmax_dev)))
      return rc;
  }
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));       // qmax is the caller's to all-reduce now
  c->match_total_rows = -1;                             // nothing to fetch or pack before the finish
  c->sopt.pending = true;
  c->sopt.p = *p;
  c->sopt.nq = nqueries;
  c->sopt.exact = exact_count;
  c->sopt.trange = find_time_range;
  c->sopt.quant = time_quantile;
  c->sopt.nrows = nrows;
  c->sopt.ranked = ranked;
  c->sopt.dq = dq;
  for (int k = 0; k < 32; ++k) c->sopt.breaks[k] = br.v[k];
  if (ranked_rows) *ranked_rows = ranked;
  return AFP_OK;
}

extern "C" int afp_match_options_shard_finish(afp_ctx* c, const int32_t* qmax_dev, int64_t* total_rows) {
  if (!c) return AFP_ERR_INVALID;
  if (!c->sopt.pending) AFP_FAIL(c, AFP_ERR_STATE, "afp_match_options_shard_rank has not been called");
  c->sopt.pending = false;
  const int nq = c->sopt.nq;
  if (nq > 0 && !qmax_dev) return AFP_ERR_INVALID;
  AFP_CUDA(c, cudaSetDevice(c->device));
  Breaks br;
  for (int k = 0; k < 32; ++k) br.v[k] = c->sopt.breaks[k];
  AFP_CUDA(c, c->d_op_qfail.reserve(sizeof(int32_t) * (size_t)std::max(nq, 1)));
  AFP_CUDA(c, cudaMemsetAsync(c->d_op_qfail.p, 0x7f, sizeof(int32_t) * (size_t)std::max(nq, 1), c->stream));
  int64_t total = 0;
  if (nq > 0 && c->sopt.p.search_depth > 0) {
    int rc = finish_options(c, c->sopt.dq, nq, c->sopt.nrows, c->sopt.ranked, &c->sopt.p, c->sopt.exact,
                            c->sopt.trange, c->sopt.quant, br, qmax_dev, c->d_op_qfail.as<int32_t>(), &total);
    if (rc) return rc;
  } else if (nq > 0) {
    AFP_CUDA(c, cudaMemsetAsync(c->d_mrow_off.p, 0, sizeof(int64_t) * (size_t)(nq + 1), c->stream));
    AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  }
  c->match_total_rows = total;
  c->sopt.finished = true;
  if (total_rows) *total_rows = total;
  return AFP_OK;
}
