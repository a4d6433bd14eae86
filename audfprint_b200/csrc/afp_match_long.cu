// K4 for long queries (whole shows, broadcast days): the general kernel's semantics spread over
// the whole grid, without its per-CTA scratch of rows x depth hits.
//
// afp_match_batch routes a query here when rows * depth >= 2^24 (AFP_LONG_HITS).  Per query, a
// sequence of grid-wide passes:
//   1. sort the rows by (bucket, time) (CUB radix sort), so that every distinct bucket is read
//      once, with the multiplicity m of its group - as the general kernel does in shared memory;
//   2. raw counts: one pass over the bucket prefixes adds m per entry to a per-id u32 counter;
//   3. candidates: every id gets the key (weight bits, id) - weight = raw / hashesperid, computed
//      as the general kernel does, 0 for ids not hit - listed in id-descending order and sorted
//      by weight descending with a stable radix sort: (weight desc, id desc), the project's tie
//      rule.  The top min(nabove, search_depth) (min(ndist, search_depth) in publish mode) are the
//      ranked candidates; no KCAP limit;
//   4. candidate hits: a second pass over the same buckets routes each hit of a row-capable
//      candidate (raw > threshcount) to that candidate's segment as dtime + bias.  A candidate's
//      raw count is exactly its segment length, so the segments are laid out by a scan of those;
//   5. modes: one CTA per candidate (grid-stride), the quick filter and candidate_modes of
//      afp_match_common.cuh over the segment, each candidate's rows into a slot of its own;
//   6. rows: the slots are compacted in rank order into the batch's row layout.
// Memory: O(nids) counters and keys, the candidates' hits, and one dense dtime histogram per CTA
// of the mode pass; nothing is sized by rows x depth.  Results do not depend on atomic order:
// raw counts and histograms are order-free and the ranking is a total order.
#include <algorithm>
#include <cub/cub.cuh>
#include "afp_match_common.cuh"

namespace {

constexpr int LT = 256;          // threads of the probe passes (one warp per bucket group)
constexpr int QF_LONG = 2048;    // segments up to this length get the quick filter before their histogram

__device__ __forceinline__ uint32_t bucket_of(unsigned long long k) { return (uint32_t)(k >> 32); }

__global__ void long_keys_kernel(const int32_t* q, int64_t n, uint32_t hmask, unsigned long long* key) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    key[i] = ((unsigned long long)((uint32_t)q[2 * i + 1] & hmask) << 32) | (uint32_t)q[2 * i];
}

// One warp per row that heads its bucket group (sorted keys): visit every live entry of the
// bucket prefix once with the group's multiplicity.  ROUTE = 0 adds m to the id's raw counter;
// ROUTE = 1 writes the m dtimes of every hit of a row-capable candidate to its segment.
template <int ROUTE>
__global__ void __launch_bounds__(LT) long_probe_kernel(MatchArgs a, const unsigned long long* key, int64_t n,
                                                        unsigned* cnt, const int32_t* slot, const int64_t* seg,
                                                        unsigned* cur, uint32_t* dts) {
  const int lane = threadIdx.x & 31;
  const uint32_t tmask = (1u << a.mtb) - 1u;
  const int64_t nwarps = (int64_t)gridDim.x * (LT / 32);
  for (int64_t r = (int64_t)blockIdx.x * (LT / 32) + (threadIdx.x >> 5); r < n; r += nwarps) {
    const uint32_t b = bucket_of(key[r]);
    if (r > 0 && bucket_of(key[r - 1]) == b) continue;        // not the head of its group (warp-uniform)
    int m = 1;
    while (r + m < n && bucket_of(key[r + m]) == b) ++m;
    const int nb = min(a.depth, a.counts[b]);
    const uint32_t* row = a.table + (size_t)b * a.depth;
    for (int s = lane; s < nb; s += 32) {
      const uint32_t v = row[s];
      const uint32_t id = (v >> a.mtb) - 1u;
      if (id >= (uint32_t)a.nids) continue;
      if (ROUTE == 0) {
        atomicAdd(&cnt[id], (unsigned)m);
      } else {
        const int j = slot[id];
        if (j < 0) continue;
        const int rt = (int)(v & tmask) + a.bias;
        const int64_t base = seg[j] + atomicAdd(&cur[j], (unsigned)m);
        for (int k = 0; k < m; ++k) dts[base + k] = (uint32_t)(rt - (int)(uint32_t)key[r + k]);
      }
    }
  }
}

// Sort input of the ranking: entry i is id nids-1-i (id descending), key = weight bits (0 = not
// hit); counts the distinct ids and those above threshcount.
__global__ void long_weights_kernel(MatchArgs a, const unsigned* cnt, unsigned long long* w, uint32_t* ids,
                                    unsigned* ndist_nabove) {
  unsigned nd = 0, na = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.nids; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t id = (uint32_t)(a.nids - 1 - i);
    const unsigned raw = cnt[id];
    w[i] = raw ? (unsigned long long)__double_as_longlong((double)raw / (double)a.hpi[id]) : 0ull;
    ids[i] = id;
    nd += raw ? 1u : 0u;
    na += raw > (unsigned)a.thresh ? 1u : 0u;
  }
  nd = __reduce_add_sync(0xffffffffu, nd);
  na = __reduce_add_sync(0xffffffffu, na);
  if ((threadIdx.x & 31) == 0 && (nd | na)) {
    atomicAdd(&ndist_nabove[0], nd);
    atomicAdd(&ndist_nabove[1], na);
  }
}

// Ranks 0..ncand-1: publish, segment length (raw count of a row-capable candidate, else 0) and
// the id -> rank map the routing pass reads.
__global__ void long_cands_kernel(MatchArgs a, int qi, int ncand, const unsigned long long* w, const uint32_t* ids,
                                  const unsigned* cnt, int32_t* slot, int32_t* seglen) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= ncand) return;
  const uint32_t id = ids[j];
  const unsigned raw = cnt[id];
  if (a.publish) {
    double* c3 = a.cand + ((size_t)qi * a.sdepth + j) * 3;
    c3[0] = (double)id;
    c3[1] = (double)raw;
    c3[2] = __longlong_as_double((long long)w[j]);
  }
  const bool rowable = raw > (unsigned)a.thresh;
  seglen[j] = rowable ? (int32_t)raw : 0;
  if (rowable) slot[id] = j;
}

// One CTA per candidate: quick filter on short segments, then the histogram-mode search.  Rank
// j's rows go to slot j of `a.rows` (a.row_cap rows each); ccnt[j] = rows it produced.
__global__ void __launch_bounds__(MT) long_modes_kernel(MatchArgs a, int ncand, const uint32_t* ids,
                                                        const int32_t* seglen, const int64_t* seg,
                                                        const uint32_t* dts, int32_t* ccnt) {
  __shared__ ModeScratch ms;
  const int tid = threadIdx.x;
  int32_t* hist = a.hist + (size_t)blockIdx.x * a.hist_len;
  int32_t* filt = a.filt + (size_t)blockIdx.x * a.hist_len;
  for (int j = blockIdx.x; j < ncand; j += gridDim.x) {
    const int n = seglen[j];
    const uint32_t* L = dts + seg[j];
    bool pass = n > 0;
    if (pass && n <= QF_LONG) {
      int best = __reduce_max_sync(0xffffffffu, max_repeat(L, n, tid, MT));
      __syncthreads();
      if ((tid & 31) == 0) ms.val[tid >> 5] = best;
      __syncthreads();
      best = 0;
      for (int w = 0; w < NW; ++w) best = max(best, ms.val[w]);
      pass = best > a.thresh;
    }
    if (pass) {
      __syncthreads();
      if (tid == 0) ms.nrows = 0;
      __syncthreads();
      candidate_modes(a, ms, hist, filt, j, n, [&](int i, int& d) { d = (int)L[i]; return true; }, ids[j], n, j);
    }
    if (tid == 0) ccnt[j] = pass ? ms.nrows : 0;
    __syncthreads();
  }
}

// One CTA: the candidates' rows in rank order -> query qi's rows of the batch, end-of-query counts.
__global__ void __launch_bounds__(MT) long_rows_kernel(MatchArgs a, int qi, int ncand, int slot_cap,
                                                       const int32_t* crows, const int32_t* ccnt, int nabove) {
  __shared__ int wsum[NW];
  const int tid = threadIdx.x;
  int done = 0;
  for (int j0 = 0; j0 < ncand; j0 += MT) {
    const int j = j0 + tid;
    const int v = j < ncand ? ccnt[j] : 0;
    const int end = block_scan_incl(v, wsum);
    const int total = wsum[NW - 1];
    const int pos = done + end - v;
    for (int k = 0; k < min(v, slot_cap) && pos + k < a.row_cap; ++k) {
      const int32_t* src = crows + ((size_t)j * slot_cap + k) * 7;
      int32_t* dst = a.rows + ((size_t)qi * a.row_cap + pos + k) * 7;
      for (int e = 0; e < 7; ++e) dst[e] = src[e];
    }
    done += total;
    __syncthreads();
  }
  if (tid == 0) query_done(a, qi, done, ncand, nabove);
}

}  // namespace

int afp_match_long(afp_ctx* c, const MatchArgs& a0, int qi, int64_t q0, int64_t nq) {
  MatchArgs a = a0;
  cudaStream_t st = c->stream;
  const int64_t nids = a.nids;
  int rc;
  // ---- 1. rows sorted by (bucket, time)
  unsigned long long *k1 = nullptr, *k2 = nullptr;
  if ((rc = afp_carve(c, c->d_lg_key, [&](Carver& k) {
         k1 = k.take<unsigned long long>(nq);
         k2 = k.take<unsigned long long>(nq);
       })) ||
      (rc = afp_launch(c, long_keys_kernel, (unsigned)std::min<int64_t>((nq + 255) / 256, 4096), 256, 0, a.q + 2 * q0,
                       nq, (1u << a.hashbits) - 1u, k1)) ||
      (rc = cub_call(c, [&](void* t, size_t& b) {
         return cub::DeviceRadixSort::SortKeys(t, b, k1, k2, (int)nq, 0, 32 + a.hashbits, st);
       })))
    return rc;
  // ---- 2. raw counts
  unsigned* cnt = nullptr;
  int32_t* slot = nullptr;
  if ((rc = afp_carve(c, c->d_lg_id, [&](Carver& k) {
         cnt = k.take<unsigned>(nids);
         slot = k.take<int32_t>(nids);
       })))
    return rc;
  unsigned* nd_na = c->d_tmp.as<unsigned>();          // (afp_match_batch reserved nqueries + 8 ints)
  AFP_CUDA(c, cudaMemsetAsync(cnt, 0, sizeof(unsigned) * (size_t)nids, st));
  AFP_CUDA(c, cudaMemsetAsync(slot, 0xff, sizeof(int32_t) * (size_t)nids, st));
  AFP_CUDA(c, cudaMemsetAsync(nd_na, 0, 2 * sizeof(unsigned), st));
  const unsigned pgrid = (unsigned)std::min<int64_t>((nq + LT / 32 - 1) / (LT / 32), (int64_t)c->num_sms * 16);
  if ((rc = afp_launch(c, long_probe_kernel<0>, pgrid, LT, 0, a, k2, nq, cnt, nullptr, nullptr, nullptr, nullptr)))
    return rc;
  // ---- 3. ranking: (weight desc, id desc)
  unsigned long long *w1 = nullptr, *w2 = nullptr;
  uint32_t *i1 = nullptr, *i2 = nullptr;
  unsigned h[2];
  if ((rc = afp_carve(c, c->d_lg_w, [&](Carver& k) {
         w1 = k.take<unsigned long long>(nids);
         w2 = k.take<unsigned long long>(nids);
         i1 = k.take<uint32_t>(nids);
         i2 = k.take<uint32_t>(nids);
       })) ||
      (rc = afp_launch(c, long_weights_kernel, (unsigned)std::min<int64_t>((nids + 255) / 256, 2048), 256, 0, a, cnt,
                       w1, i1, nd_na)) ||
      (rc = cub_call(c, [&](void* t, size_t& b) {
         return cub::DeviceRadixSort::SortPairsDescending(t, b, w1, w2, i1, i2, (int)nids, 0, 64, st);
       })) ||
      (rc = afp_read_back(c, h, nd_na, 2)))
    return rc;
  const int ndist = (int)h[0], nabove = (int)h[1];
  const int ncand = a.publish ? std::min(ndist, a.sdepth) : std::min(nabove, a.sdepth);
  // ---- 4. candidate segments and their hits
  const int slot_cap = std::max(1, std::min(a.maxalign + 1, a.row_cap));
  int64_t* seg = nullptr;
  int32_t *seglen = nullptr, *ccnt = nullptr, *crows = nullptr;
  unsigned* cur = nullptr;
  if ((rc = afp_carve(c, c->d_lg_cand, [&](Carver& k) {
         seg = k.take<int64_t>(ncand + 1);
         seglen = k.take<int32_t>(ncand + 1);
         cur = k.take<unsigned>(ncand + 1);
         ccnt = k.take<int32_t>(ncand + 1);
         crows = k.take<int32_t>(7 * (int64_t)ncand * slot_cap);
       })))
    return rc;
  if (ncand > 0) {
    int64_t nseg = 0;
    if ((rc = afp_launch(c, long_cands_kernel, (ncand + 255) / 256, 256, 0, a, qi, ncand, w2, i2, cnt, slot, seglen)) ||
        (rc = afp_launch_scan_i32_to_i64(c, seglen, seg, ncand)) || (rc = afp_read_back(c, &nseg, seg + ncand, 1)))
      return rc;
    AFP_CUDA(c, c->d_lg_dts.reserve(sizeof(uint32_t) * (size_t)(nseg + 1)));
    uint32_t* dts = c->d_lg_dts.as<uint32_t>();
    AFP_CUDA(c, cudaMemsetAsync(cur, 0, sizeof(unsigned) * (size_t)ncand, st));
    if (nseg > 0 && (rc = afp_launch(c, long_probe_kernel<1>, pgrid, LT, 0, a, k2, nq, nullptr, slot, seg, cur, dts)))
      return rc;
    // ---- 5. modes, one CTA per candidate; each rank's rows go to a slot of its own
    MatchArgs am = a;
    am.rows = crows;
    am.row_cap = slot_cap;
    if ((rc = afp_launch(c, long_modes_kernel, std::min(ncand, c->lg_ctas), MT, 0, am, ncand, i2, seglen, seg, dts,
                         ccnt)))
      return rc;
  }
  // ---- 6. rows in rank order, end-of-query counts
  return afp_launch(c, long_rows_kernel, 1, MT, 0, a, qi, ncand, slot_cap, crows, ccnt, nabove);
}
