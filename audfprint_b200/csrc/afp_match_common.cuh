// Pieces shared by the matching kernels (afp_match.cu: general path, afp_match_fast.cu: fast path;
// afp_match_long.cu reuses the quick filter and the mode search): kernel arguments and the fast kernel's launcher, launch geometry, candidate order,
// block-wide helpers (scan, bitonic sort, arg-max) and the candidate stage that follows the
// ranking in both kernels - publish and dt-list offsets of the top-K, quick filter, per-candidate
// dtime histogram and its mode search (audfprint_match.py:284-311), end-of-query counts.  Each
// kernel finds its ranked candidates and routes their hits to the dt lists in its own way.
#pragma once
#include <math.h>
#include "afp_internal.cuh"

struct MatchArgs {
  const int32_t* q;        // [sum nq][2]
  const int64_t* qoff;     // [nq+1] (device)
  int nqueries;
  const uint32_t* table;
  const int32_t* counts;
  const uint32_t* hpi;
  int hashbits, depth, mtb;
  int64_t nids;
  int window, thresh, sdepth, maxalign;
  // per-CTA scratch (stride in elements)
  uint2* hits;      int64_t hits_cap;     // (id, dt + bias)
  uint32_t* dlist;                        // distinct ids, hits_cap
  double* wtd;                            // weighted count per dlist entry, hits_cap
  uint32_t* dts;                          // dt + bias of the candidates' hits, grouped per candidate, hits_cap
  uint32_t* recs;                         // (id << 8 | weight) of every distinct (bucket, slot), hits_cap
  uint32_t* rawl;                         // raw count per dlist entry, hits_cap
  int32_t* hist;    int hist_len;         // dtime histogram
  int32_t* filt;                          // local-max filtered copy
  int bias;
  int32_t* rows;    int row_cap;          // [nqueries][row_cap][7]
  int32_t* row_cnt;                       // [nqueries] rows produced (may exceed row_cap)
  // sharded-table mode: publish every query's local top-sdepth candidate list
  int publish;                            // 0/1
  double* cand;                           // [nqueries][sdepth][3] = (id, raw, weight)
  int32_t* cand_cnt;                      // [nqueries][2] = (entries, n_above)
  // work list of the general kernel (NULL = every query); the fast kernel appends the queries
  // it hands over (capacity overflow, parameters outside its limits)
  int32_t* qlist;
  int* nlist;
  int32_t* fstat;                         // [nqueries] 0 = done by the fast kernel, else the reason it was not
  const unsigned char* qskip;             // [nqueries] 1 = long query (afp_match_long.cu), not the fast kernel's; NULL = none
  // fast path (afp_match_fast.cu)
  uint2* mhits;     int mh_cap;           // per-CTA list of the hits of multi-record ids: (set slot, dt + bias)
  unsigned hmin;                          // smallest hashesperid of the table; 0 = unknown (no pruning)
  int bm_exact;                           // nids <= bitmap bits: the repeat bitmap is indexed by the id itself
};

// The fast kernel over every query (afp_match_fast.cu); it appends the ones it hands over to a.qlist.
cudaError_t afp_launch_match_fast(const MatchArgs& a, int nctas, cudaStream_t stream);
// Query qi (rows q0 .. q0+nq of a.q) on the long-query path (afp_match_long.cu): writes its rows,
// row count and, in publish mode, its candidate list.  a.hist / a.filt / a.hist_len / a.bias are
// the mode pass's per-CTA histograms (zeroed; left zeroed), c->lg_ctas CTAs of them.
int afp_match_long(afp_ctx* c, const MatchArgs& a, int qi, int64_t q0, int64_t nq);
// rows * depth from which a query takes the long-query path
constexpr int64_t AFP_LONG_HITS = (int64_t)1 << 24;

namespace {

constexpr int MT = 1024;          // threads per matching CTA (one CTA per SM, persistent over the queries)
constexpr int NW = MT / 32;
constexpr int KCAP = 1024;        // candidate depth handled by the fast path (search_depth <= KCAP)

// candidate order: (weighted count desc, id desc); keys are (bits of the positive double, id)
__device__ __forceinline__ bool key_gt(unsigned long long w1, unsigned i1, unsigned long long w2, unsigned i2) {
  return w1 > w2 || (w1 == w2 && i1 > i2);
}

// scratch the block-wide helpers need, embedded in each kernel's shared-memory struct
struct ModeScratch {
  int val[NW], idx[NW];
  int nrows;
  int dmin, dmax;
};

// The ranked candidates of one query in shared memory, index = rank: id, raw count, and the
// start, fill cursor and quick-filter verdict of each candidate's dt list.
struct CandArrays {
  const unsigned* id;
  const unsigned* raw;
  int* loff;
  int* cur;
  unsigned char* pass;
};

// 96-bit composite key (weight bits, id), 12 digits of 8 bits from the top
__device__ __forceinline__ unsigned key_digit(unsigned long long w, unsigned id, int p) {
  return p < 8 ? (unsigned)(w >> (56 - 8 * p)) & 0xffu : (id >> (24 - 8 * (p - 8))) & 0xffu;
}
// compare the top `nfix` digits of (w,id) with those of the prefix: -1 below, 0 equal, +1 above
__device__ __forceinline__ int prefix_cmp(unsigned long long w, unsigned id, unsigned long long pw, unsigned pid,
                                          int nfix) {
  if (nfix == 0) return 0;
  if (nfix <= 8) {
    const int sh = 64 - 8 * nfix;
    const unsigned long long a = w >> sh, b = pw >> sh;
    return a > b ? 1 : (a < b ? -1 : 0);
  }
  if (w != pw) return w > pw ? 1 : -1;
  const int sh = 32 - 8 * (nfix - 8);
  const unsigned a = sh ? id >> sh : id, b = sh ? pid >> sh : pid;
  return a > b ? 1 : (a < b ? -1 : 0);
}

// inclusive scan of one int per thread over the CTA (MT threads)
__device__ __forceinline__ int block_scan_incl(int v, int* wsum) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  __syncthreads();
  if (lane == 31) wsum[warp] = v;
  __syncthreads();
  if (warp == 0) {
    int w = wsum[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += t;
    }
    wsum[lane] = w;
  }
  __syncthreads();
  return v + (warp ? wsum[warp - 1] : 0);
}

// Block-wide bitonic network over n2 entries (a power of two): entries i < l of a stage whose
// sorted runs are k long are exchanged by swap(i, l) when out_of_order(i, l, k).
template <class OutOfOrder, class Swap>
__device__ __forceinline__ void bitonic_sort(int n2, OutOfOrder out_of_order, Swap swap) {
  for (int k = 2; k <= n2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n2; i += MT) {
        const int l = i ^ j;
        if (l > i && out_of_order(i, l, k)) swap(i, l);
      }
      __syncthreads();
    }
}

// (value desc, index asc) arg-max over f[lo..hi] == np.argmax (first max)
__device__ inline void block_argmax(const int32_t* f, int lo, int hi, ModeScratch& sh, int& best_v, int& best_i) {
  const int tid = threadIdx.x;
  int v = -1, ix = 0x7fffffff;
  for (int i = lo + tid; i <= hi; i += MT) {
    const int x = f[i];
    if (x > v) { v = x; ix = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const int ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, ix, o);
    if (ov > v || (ov == v && oi < ix)) { v = ov; ix = oi; }
  }
  __syncthreads();
  if ((tid & 31) == 0) { sh.val[tid >> 5] = v; sh.idx[tid >> 5] = ix; }
  __syncthreads();
  best_v = sh.val[0];
  best_i = sh.idx[0];
  for (int w = 1; w < NW; ++w)
    if (sh.val[w] > best_v || (sh.val[w] == best_v && sh.idx[w] < best_i)) { best_v = sh.val[w]; best_i = sh.idx[w]; }
}

// One candidate of query qi: its dense dtime histogram from n entries - dt(i, d) stores entry i's
// dtime in d and says whether the entry belongs to the candidate - then the histogram-mode search
// (audfprint_match.py:284-311).  Emits rows, restores hist to zero.
template <class Dt>
__device__ inline void candidate_modes(const MatchArgs& a, ModeScratch& sh, int32_t* hist, int32_t* filt, int qi, int n,
                                       Dt dt, unsigned id, int raw, int rank) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { sh.dmin = 0x7fffffff; sh.dmax = -1; }
  __syncthreads();
  {
    int dmin = 0x7fffffff, dmax = -1;
    for (int i = tid; i < n; i += MT) {
      int d;
      if (dt(i, d)) {
        atomicAdd(&hist[d], 1);
        dmin = min(dmin, d);
        dmax = max(dmax, d);
      }
    }
    dmin = __reduce_min_sync(0xffffffffu, dmin);
    dmax = __reduce_max_sync(0xffffffffu, dmax);
    if (lane == 0 && dmax >= 0) { atomicMin(&sh.dmin, dmin); atomicMax(&sh.dmax, dmax); }
  }
  __syncthreads();
  const int lo = sh.dmin, hi = sh.dmax;
  // keep_local_maxes (:70-75, locmax :51-67); zero-extended ends are equivalent
  for (int i = lo + tid; i <= hi; i += MT) {
    const int v = __ldcg(hist + i), l = __ldcg(hist + i - 1), r = __ldcg(hist + i + 1);
    filt[i] = (v >= l && r < v) ? v : 0;
  }
  __syncthreads();
  int found = 0;
  while (true) {
    int bv, bi;
    block_argmax(filt, lo, hi, sh, bv, bi);   // :290 np.argmax = first max
    if (bv <= a.thresh) break;                // :291
    // :295 count over +-window (hist is zero outside the touched range)
    int part = 0;
    for (int t2 = tid; t2 <= 2 * a.window; t2 += MT) part += __ldcg(hist + bi - a.window + t2);
    part = __reduce_add_sync(0xffffffffu, part);
    __syncthreads();
    if (lane == 0) sh.val[warp] = part;
    __syncthreads();
    if (tid == 0) {
      int count = 0;
      for (int w = 0; w < NW; ++w) count += sh.val[w];
      const int nr = sh.nrows;
      if (nr < a.row_cap) {
        int32_t* row = a.rows + ((size_t)qi * a.row_cap + nr) * 7;
        row[0] = (int32_t)id; row[1] = count; row[2] = bi - a.bias; row[3] = raw;
        row[4] = rank; row[5] = 0; row[6] = 0;                      // :300-301
      }
      sh.nrows = nr + 1;
    }
    for (int t2 = tid; t2 <= 2 * a.window; t2 += MT) {              // :307-308
      const int i = bi - a.window + t2;
      if (i >= lo && i <= hi) filt[i] = 0;
    }
    __syncthreads();
    ++found;
    if (found > a.maxalign) break;                                   // :309-311
  }
  __syncthreads();
  for (int i = lo + tid; i <= hi; i += MT) hist[i] = 0;              // restore the scratch
  __syncthreads();
}

// Quick filter of a candidate's dt list L[0..n): the largest number of times one of the entries
// i0, i0 + step, ... occurs in the list (the caller reduces over the threads that split it).  The
// largest dtime bin is the maximum over all entries; a row needs it above threshcount (:291).
__device__ __forceinline__ int max_repeat(const uint32_t* L, int n, int i0, int step) {
  int best = 0;
  for (int i = i0; i < n; i += step) {
    const uint32_t me = L[i];
    int cnt = 0;
    for (int k = 0; k < n; ++k) cnt += (L[k] == me) ? 1 : 0;
    best = max(best, cnt);
  }
  return best;
}

// Start of the candidate stage: thread `tid` < ncand holds rank tid's (id, raw, weight bits).
// Publishes the ranked list in shard mode and lays out the dt lists of the candidates that can
// yield rows (raw > threshcount, :291) back to back; returns whether rank tid is one of them.
__device__ __forceinline__ bool candidates_begin(const MatchArgs& a, int qi, int ncand, unsigned id, unsigned raw,
                                                 unsigned long long wb, const CandArrays& c, int* wsum) {
  const int tid = threadIdx.x;
  const bool rowable = tid < ncand && raw > (unsigned)a.thresh;
  const int lraw = rowable ? (int)raw : 0;
  const int lend = block_scan_incl(lraw, wsum);
  if (tid < ncand) {
    if (a.publish) {
      double* c3 = a.cand + ((size_t)qi * a.sdepth + tid) * 3;
      c3[0] = (double)id;
      c3[1] = (double)raw;
      c3[2] = __longlong_as_double((long long)wb);
    }
    c.loff[tid] = lend - lraw;
    c.cur[tid] = 0;
    c.pass[tid] = 0;
  }
  return rowable;
}

// End of the candidate stage, once the caller has routed the hits to the dt lists: quick filter,
// then the full mode search of the surviving candidates in rank order.
__device__ __forceinline__ void candidates_finish(const MatchArgs& a, int qi, int ncand, const CandArrays& c,
                                                  const uint32_t* dts, ModeScratch& ms, int32_t* hist, int32_t* filt) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // quick filter, one warp per candidate: a row needs a dtime bin > threshcount (:291)
  for (int j = warp; j < ncand; j += NW) {
    const int n = (int)c.raw[j];
    if (n <= a.thresh) continue;       // warp-uniform
    const int best = __reduce_max_sync(0xffffffffu, max_repeat(dts + c.loff[j], n, lane, 32));
    if (lane == 0) c.pass[j] = best > a.thresh;
  }
  __syncthreads();
  for (int j = 0; j < ncand; ++j) {
    if (!c.pass[j]) continue;          // uniform
    const int n = (int)c.raw[j];
    const uint32_t* L = dts + c.loff[j];
    candidate_modes(a, ms, hist, filt, qi, n, [&](int i, int& d) { d = (int)L[i]; return true; }, c.id[j], n, j);
  }
}

// a query's row count and, in shard mode, its candidate counts (one thread)
__device__ __forceinline__ void query_done(const MatchArgs& a, int qi, int nrows, int ncand, int nabove) {
  a.row_cnt[qi] = nrows;
  if (a.publish) {
    a.cand_cnt[2 * qi] = ncand;
    a.cand_cnt[2 * qi + 1] = nabove;
  }
}

}  // namespace
