// K4 — device-resident hash table: bucket probe, per-track raw counts,
// weighted candidate ranking and per-candidate time-offset histogram modes.
//
// Replaces HashTable.get_hits (hash_table.py:150-176),
// Matcher._best_count_ids (audfprint_match.py:124-147) and
// Matcher._approx_match_counts (:241-312, find_time_range off).
//
// One 1024-thread CTA per query (persistent over the batch, one per SM).  Each CTA
// owns a private scratch region in HBM (hit list, records, distinct-id list, dense
// dtime histogram cleared over the touched range); the per-track raw counts are
// built in shared memory, segment by segment.  Results do not depend on hit
// order, so hits and records are appended with (shared-memory) atomics.
// Once the candidates are ranked and their hits routed, the candidate stage
// (quick filter, dtime histograms, modes) is the fast kernel's, from
// afp_match_common.cuh.
//
// Tie rule (documented deviation, see oracle/afp_oracle.py::rank_candidates):
// the reference reverses an unstable argsort, so the order of equal weighted
// counts is implementation-defined there; here it is (weight desc, id desc).
#include <math.h>
#include <algorithm>
#include "afp_match_common.cuh"

namespace {

constexpr int GCAP = 1024;        // radix select stops once the undecided set is this small
constexpr int QCAP = 16384;       // query rows sorted in shared memory to merge probes of one bucket (128 KB)
constexpr int CSEG = 32768;       // track ids counted per pass in shared memory (u32 counters, the same 128 KB)
constexpr int64_t HITS_MAX = (int64_t)1 << 30;   // per-query hit capacity (rows * depth): int indexing
constexpr int HSET_BITS = 11;     // candidate hash set: 2048 entries for <= KCAP = 1024 keys
constexpr int HSET = 1 << HSET_BITS;

struct Shared {
  ModeScratch ms;
  unsigned long long a_w[KCAP + GCAP];   // gathered keys, sorted descending: the top-K' candidates
  unsigned a_id[KCAP + GCAP];
  unsigned a_raw[KCAP];
  int loff[KCAP];        // start of candidate j's dt list
  int cur[KCAP];         // fill cursor of candidate j's dt list
  unsigned char pass[KCAP];
  int rhist[256];        // radix-select digit histogram
  int wsum[NW];
  unsigned long long kw[NW];
  unsigned kid[NW];
  unsigned nhits, ndist, nabove, ngather, nrec;
  int sel_digit, sel_need, sel_m;
  int segoff[514];       // record range of every id segment (nids < 2^24 -> <= 512 segments)
  int segcur[512];
};

// raw count of a selected id from its weight: w = raw / hpi correctly rounded, so
// rint(w * hpi) == raw exactly (raw < 2^21).  hashesperid == 0 (w = inf) falls back to a scan.
__device__ __forceinline__ unsigned raw_of(const MatchArgs& a, unsigned long long wbits, unsigned id,
                                           const uint32_t* dlist, const uint32_t* rawl, int ndist) {
  const unsigned h = a.hpi[id];
  if (h != 0u) return __double2uint_rn(__longlong_as_double((long long)wbits) * (double)h);
  for (int i = 0; i < ndist; ++i)
    if (dlist[i] == id) return rawl[i];
  return 0u;
}

__global__ void __launch_bounds__(MT) afp_match_kernel(MatchArgs a) {
  __shared__ Shared sh;
  extern __shared__ unsigned long long s_q[];   // QCAP (bucket << 32 | query time) keys
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint2* hits = a.hits + (size_t)blockIdx.x * a.hits_cap;
  uint32_t* dlist = a.dlist + (size_t)blockIdx.x * a.hits_cap;
  double* wtd = a.wtd + (size_t)blockIdx.x * a.hits_cap;
  uint32_t* dts = a.dts + (size_t)blockIdx.x * a.hits_cap;
  uint32_t* recs = a.recs + (size_t)blockIdx.x * a.hits_cap;
  uint32_t* rawl = a.rawl + (size_t)blockIdx.x * a.hits_cap;
  unsigned* s_cnt = reinterpret_cast<unsigned*>(s_q);   // CSEG counters, aliases the sorted query rows
  int32_t* hist = a.hist + (size_t)blockIdx.x * a.hist_len;
  int32_t* filt = a.filt + (size_t)blockIdx.x * a.hist_len;
  const uint32_t hmask = (1u << a.hashbits) - 1u, tmask = (1u << a.mtb) - 1u;
  for (int i = tid; i < CSEG / 4; i += MT) reinterpret_cast<uint4*>(s_cnt)[i] = make_uint4(0u, 0u, 0u, 0u);
  __syncthreads();

  // every query, or the ones the fast kernel handed over (afp_match_fast.cu)
  const int nwork = a.qlist ? *a.nlist : a.nqueries;
  for (int wk = blockIdx.x; wk < nwork; wk += gridDim.x) {
    const int qi = a.qlist ? a.qlist[wk] : wk;
    const int64_t q0 = a.qoff[qi];
    const int nq = (int)(a.qoff[qi + 1] - q0);
    if (tid == 0) { sh.nhits = 0; sh.ndist = 0; sh.nabove = 0; sh.ms.nrows = 0; sh.nrec = 0; }
    __syncthreads();
    // ---- probe (hash_table.py:162-173).  A query made of several sub-frame shifts probes
    // the same bucket up to `shifts` times (same hash at neighbouring times): the rows are
    // sorted by bucket in shared memory so that every distinct bucket is read ONCE and every
    // (bucket, id) pair costs ONE counter atomic of weight m.  Hit order is irrelevant
    // downstream (raw counts and dtime histograms are order-free).
    const bool sorted = nq <= QCAP;
    int n2 = 1;
    if (sorted) {
      while (n2 < nq) n2 <<= 1;
      for (int i = tid; i < n2; i += MT)
        s_q[i] = i < nq ? ((unsigned long long)((uint32_t)a.q[2 * (q0 + i) + 1] & hmask) << 32) |
                              (uint32_t)a.q[2 * (q0 + i)]
                        : ~0ull;
      __syncthreads();
      bitonic_sort(                              // ascending (bucket, time)
          n2, [&](int i, int l, int k) { return (s_q[i] > s_q[l]) == ((i & k) == 0); },
          [&](int i, int l) { const unsigned long long x = s_q[i]; s_q[i] = s_q[l]; s_q[l] = x; });
    }
    for (int r = warp; r < nq; r += NW) {
      uint32_t b;
      int m = 1, qt0 = 0;
      if (sorted) {
        const unsigned long long e = s_q[r];
        b = (uint32_t)(e >> 32);
        if (r > 0 && (uint32_t)(s_q[r - 1] >> 32) == b) continue;      // not the head of its bucket group
        while (r + m < nq && (uint32_t)(s_q[r + m] >> 32) == b) ++m;
      } else {
        qt0 = a.q[2 * (q0 + r)];
        b = (uint32_t)a.q[2 * (q0 + r) + 1] & hmask;
      }
      const int n = min(a.depth, a.counts[b]);
      const uint32_t* row = a.table + (size_t)b * a.depth;
      for (int s0 = 0; s0 < n; s0 += 128) {
        uint32_t v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = (s0 + 32 * u + lane < n) ? row[s0 + 32 * u + lane] : 0u;
        const int chunk = min(128, n - s0);
        unsigned basepos = 0;
        if (lane == 0) basepos = atomicAdd(&sh.nhits, (unsigned)(chunk * m));
        basepos = __shfl_sync(0xffffffffu, basepos, 0);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          bool rec = false;
          uint32_t id = 0;
          if (s0 + 32 * u + lane < n) {
            id = (v[u] >> a.mtb) - 1u;
            const int rt = (int)(v[u] & tmask) + a.bias;
            for (int k = 0; k < m; ++k) {
              const int qt = sorted ? (int)(uint32_t)s_q[r + k] : qt0;
              hits[basepos + k * chunk + 32 * u + lane] = make_uint2(id, (unsigned)(rt - qt));
            }
            rec = id < (uint32_t)a.nids;
          }
          // one record (id, weight m) per distinct (bucket, slot): the raw counts are built
          // from these in shared memory, no global atomics
          const unsigned rm = __ballot_sync(0xffffffffu, rec);
          const int per = (m + 254) / 255;                       // weights above 255 are split
          if (rm) {
            unsigned base = 0;
            if (lane == 0) base = atomicAdd(&sh.nrec, (unsigned)(__popc(rm) * per));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (rec) {
              uint32_t* dst = recs + base + __popc(rm & ((1u << lane) - 1u)) * per;
              for (int k = 0, left = m; k < per; ++k, left -= 255) dst[k] = (id << 8) | (uint32_t)min(left, 255);
            }
          }
        }
      }
    }
    __syncthreads();
    // ---- raw count per track and weighted counts (audfprint_match.py:129-144): the ids are
    // swept in segments of CSEG, each counted in shared memory (the 128 KB that held the
    // sorted query rows), then every non-zero counter becomes a distinct-list entry
    {
      const int nrec = (int)sh.nrec;
      const int nseg = (int)((a.nids + CSEG - 1) / CSEG);        // <= 512 (nids < 2^24)
      // group the records by id segment (counting sort: histogram, scan, scatter into `dts`)
      // so that each counting pass reads only its own records instead of all of them
      for (int i = tid; i <= nseg; i += MT) sh.segoff[i] = 0;
      __syncthreads();
      for (int i0 = 0; i0 < nrec; i0 += 4 * MT) {
        uint32_t rr[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) rr[u] = (i0 + u * MT + tid < nrec) ? recs[i0 + u * MT + tid] : 0xffffffffu;
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (rr[u] != 0xffffffffu) atomicAdd(&sh.segoff[(rr[u] >> 8) / CSEG + 1], 1);
      }
      __syncthreads();
      if (tid == 0)
        for (int i = 1; i <= nseg; ++i) sh.segoff[i] += sh.segoff[i - 1];
      __syncthreads();
      for (int i = tid; i < nseg; i += MT) sh.segcur[i] = sh.segoff[i];
      __syncthreads();
      for (int i0 = 0; i0 < nrec; i0 += 4 * MT) {
        uint32_t rr[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) rr[u] = (i0 + u * MT + tid < nrec) ? recs[i0 + u * MT + tid] : 0xffffffffu;
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (rr[u] != 0xffffffffu) dts[atomicAdd(&sh.segcur[(rr[u] >> 8) / CSEG], 1)] = rr[u];
      }
      __syncthreads();
      // the counters must start from zero: clear what the sorted query rows occupied (every
      // pass below leaves the array zeroed again)
      {
        uint4* z4 = reinterpret_cast<uint4*>(s_cnt);
        // n2 keys of 8 bytes = n2/2 uint4, at least one (a 0- or 1-row query leaves one key); an
        // unsorted query wrote nothing here and finds the zeros the previous harvest left
        const int nz = sorted ? max(1, n2 / 2) : 0;
        for (int i = tid; i < nz; i += MT) z4[i] = make_uint4(0u, 0u, 0u, 0u);
      }
      __syncthreads();
      unsigned above = 0;
      for (int sg = 0; sg < nseg; ++sg) {
        const int r0 = sh.segoff[sg], r1 = sh.segoff[sg + 1];
        if (r1 == r0) continue;                                   // uniform: no id of this segment was hit
        const uint32_t seg0 = (uint32_t)sg * CSEG;
        for (int i = r0 + tid; i < r1; i += MT) {
          const uint32_t rr = dts[i];
          atomicAdd(&s_cnt[(rr >> 8) - seg0], rr & 255u);
        }
        __syncthreads();
        // harvest through the records again: whoever swaps a non-zero counter out owns that id;
        // the array is all-zero afterwards (no scan of 32768 counters, no re-zeroing)
        for (int i0 = r0; i0 < r1; i0 += MT) {
          const int i = i0 + tid;
          unsigned raw = 0, id = 0;
          if (i < r1) {
            id = dts[i] >> 8;
            raw = atomicExch(&s_cnt[id - seg0], 0u);
          }
          const unsigned hm = __ballot_sync(0xffffffffu, raw != 0u);
          if (hm) {
            unsigned base = 0;
            if (lane == 0) base = atomicAdd(&sh.ndist, (unsigned)__popc(hm));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (raw) {
              const unsigned pos = base + __popc(hm & ((1u << lane) - 1u));
              dlist[pos] = id;
              rawl[pos] = raw;
              wtd[pos] = (double)raw / (double)a.hpi[id];
              above += raw > (uint32_t)a.thresh ? 1u : 0u;
            }
          }
        }
        __syncthreads();
      }
      above = __reduce_add_sync(0xffffffffu, above);
      if (lane == 0 && above) atomicAdd(&sh.nabove, above);
    }
    __syncthreads();
    __syncthreads();
    const int nhits = (int)sh.nhits, ndist = (int)sh.ndist;
    const int nabove = (int)sh.nabove;
    // candidate depth: min(#ids above threshold, search_depth) (:142-144); a table shard
    // publishes its full local top-search_depth list instead (dist.merge_sharded_results)
    const int maxdepth = a.publish ? min(ndist, a.sdepth) : min(nabove, a.sdepth);

    if (maxdepth > 0 && maxdepth <= KCAP) {
      // ---- fast path: the top-`maxdepth` distinct ids by (weight desc, id desc) via an
      // MSB-first radix select on the 96-bit key, stopped as soon as the undecided set fits
      // in shared memory, then one small bitonic sort.  Position in the sorted list = rank.
      unsigned long long pw = 0ull;
      unsigned pid = 0u;
      int nfix = 0, need = maxdepth, m = ndist;
      while (m > GCAP && nfix < 12) {
        for (int i = tid; i < 256; i += MT) sh.rhist[i] = 0;
        __syncthreads();
        for (int i0 = 0; i0 < ndist; i0 += 4 * MT) {
          unsigned long long w4[4];
          unsigned id4[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int i = i0 + u * MT + tid;
            w4[u] = i < ndist ? (unsigned long long)__double_as_longlong(wtd[i]) : 0ull;
            id4[u] = i < ndist ? dlist[i] : 0u;
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            int d = -1;
            if (i0 + u * MT + tid < ndist && prefix_cmp(w4[u], id4[u], pw, pid, nfix) == 0)
              d = (int)key_digit(w4[u], id4[u], nfix);
            const unsigned peers = __match_any_sync(0xffffffffu, d);   // warp-aggregated histogram
            if (d >= 0 && lane == __ffs(peers) - 1) atomicAdd(&sh.rhist[d], __popc(peers));
          }
        }
        __syncthreads();
        if (tid == 0) {
          int cum = 0, b = 255;
          for (; b > 0; --b) {
            if (cum + sh.rhist[b] >= need) break;
            cum += sh.rhist[b];
          }
          sh.sel_digit = b;
          sh.sel_need = need - cum;
          sh.sel_m = sh.rhist[b];
        }
        __syncthreads();
        const unsigned dg = (unsigned)sh.sel_digit;
        if (nfix < 8) pw |= (unsigned long long)dg << (56 - 8 * nfix); else pid |= dg << (24 - 8 * (nfix - 8));
        need = sh.sel_need;
        m = sh.sel_m;
        ++nfix;
        __syncthreads();
      }
      if (tid == 0) sh.ngather = 0;
      __syncthreads();
      for (int i0 = 0; i0 < ndist; i0 += MT) {     // gather: decided-in ids + the undecided set
        const int i = i0 + tid;
        bool take = false;
        unsigned long long w = 0ull;
        unsigned id = 0u;
        if (i < ndist) {
          w = (unsigned long long)__double_as_longlong(wtd[i]);
          id = dlist[i];
          take = prefix_cmp(w, id, pw, pid, nfix) >= 0;
        }
        const unsigned tm = __ballot_sync(0xffffffffu, take);
        if (tm) {
          unsigned base = 0;
          if (lane == 0) base = atomicAdd(&sh.ngather, (unsigned)__popc(tm));
          base = __shfl_sync(0xffffffffu, base, 0);
          if (take) {
            const unsigned pos = base + __popc(tm & ((1u << lane) - 1u));
            sh.a_w[pos] = w;
            sh.a_id[pos] = id;
          }
        }
      }
      __syncthreads();
      const int ng = (int)sh.ngather;           // maxdepth <= ng <= maxdepth - need + m <= KCAP + GCAP
      int n2 = 1;
      while (n2 < ng) n2 <<= 1;
      for (int i = ng + tid; i < n2; i += MT) { sh.a_w[i] = 0ull; sh.a_id[i] = 0u; }
      __syncthreads();
      bitonic_sort(                              // descending
          n2, [&](int i, int l, int k) { return key_gt(sh.a_w[i], sh.a_id[i], sh.a_w[l], sh.a_id[l]) != ((i & k) == 0); },
          [&](int i, int l) {
            const unsigned long long tw = sh.a_w[i]; sh.a_w[i] = sh.a_w[l]; sh.a_w[l] = tw;
            const unsigned ti = sh.a_id[i]; sh.a_id[i] = sh.a_id[l]; sh.a_id[l] = ti;
          });
      const int ncand = maxdepth;               // entries 0..maxdepth-1 of the sorted list, rank = index
      const CandArrays cands{sh.a_id, sh.a_raw, sh.loff, sh.cur, sh.pass};
      {
        unsigned id = 0, raw = 0;
        unsigned long long wb = 0ull;
        if (tid < ncand) {
          id = sh.a_id[tid];
          wb = sh.a_w[tid];
          raw = raw_of(a, wb, id, dlist, rawl, ndist);
          sh.a_raw[tid] = raw;
        }
        const bool rowable = candidates_begin(a, qi, ncand, id, raw, wb, cands, sh.wsum);
        // id -> candidate slot: open-addressing hash set in the (now free) upper halves of the
        // sort arrays, so that routing the hits costs no global access
        unsigned* hkey = reinterpret_cast<unsigned*>(sh.a_w + KCAP);              // HSET entries
        unsigned short* hval = reinterpret_cast<unsigned short*>(sh.a_id + KCAP);
        for (int i = tid; i < HSET; i += MT) hkey[i] = 0u;
        __syncthreads();
        if (rowable) {
          const unsigned key = id + 1u;
          unsigned h = (id * 2654435761u) >> (32 - HSET_BITS);
          while (atomicCAS(&hkey[h], 0u, key) != 0u) h = (h + 1u) & (HSET - 1);
          hval[h] = (unsigned short)tid;
        }
        __syncthreads();
        // ---- one pass over the hits: route the hits of candidates to their dt lists
        for (int i0 = 0; i0 < nhits; i0 += 4 * MT) {
          uint2 h4[4];
#pragma unroll
          for (int u = 0; u < 4; ++u)
            h4[u] = (i0 + u * MT + tid < nhits) ? hits[i0 + u * MT + tid] : make_uint2(0xffffffffu, 0u);
#pragma unroll
          for (int u = 0; u < 4; ++u) {
          const uint2 hh = h4[u];
          if (hh.x == 0xffffffffu) continue;
          const unsigned key = hh.x + 1u;
          unsigned h = (hh.x * 2654435761u) >> (32 - HSET_BITS);
          unsigned k;
          while ((k = hkey[h]) != 0u) {
            if (k == key) {
              const int slot = hval[h];
              dts[sh.loff[slot] + atomicAdd(&sh.cur[slot], 1)] = hh.y;
              break;
            }
            h = (h + 1u) & (HSET - 1);
          }
          }
        }
      }
      __syncthreads();
      candidates_finish(a, qi, ncand, cands, dts, sh.ms, hist, filt);
    } else if (maxdepth > 0) {
      // ---- slow path (search_depth > KCAP): one pass over the distinct
      // ids and one over the hits per candidate
      unsigned long long pw = ~0ull;
      unsigned pid = ~0u;
      bool have_prev = false;
      for (int rank = 0; rank < maxdepth; ++rank) {
        unsigned long long bw = 0ull;
        unsigned bid = 0u;
        bool bvld = false;
        for (int i = tid; i < ndist; i += MT) {
          const unsigned long long w = (unsigned long long)__double_as_longlong(wtd[i]);
          const unsigned id = dlist[i];
          if (have_prev && !key_gt(pw, pid, w, id)) continue;
          if (!bvld || key_gt(w, id, bw, bid)) { bw = w; bid = id; bvld = true; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const unsigned long long ow = __shfl_xor_sync(0xffffffffu, bw, o);
          const unsigned oid = __shfl_xor_sync(0xffffffffu, bid, o);
          const bool ov = __shfl_xor_sync(0xffffffffu, (int)bvld, o) != 0;
          if (ov && (!bvld || key_gt(ow, oid, bw, bid))) { bw = ow; bid = oid; bvld = true; }
        }
        __syncthreads();
        if (lane == 0) { sh.kw[warp] = bw; sh.kid[warp] = bid; sh.ms.val[warp] = bvld; }
        __syncthreads();
        bvld = false;
        for (int w = 0; w < NW; ++w)
          if (sh.ms.val[w] && (!bvld || key_gt(sh.kw[w], sh.kid[w], bw, bid))) { bw = sh.kw[w]; bid = sh.kid[w]; bvld = true; }
        if (!bvld) break;
        pw = bw; pid = bid; have_prev = true;
        const int raw = (int)raw_of(a, bw, bid, dlist, rawl, ndist);
        if (a.publish) {
          double* c3 = a.cand + ((size_t)qi * a.sdepth + rank) * 3;
          if (tid == 0) { c3[0] = (double)bid; c3[1] = (double)raw; c3[2] = __longlong_as_double((long long)bw); }
        }
        if (raw <= a.thresh) continue;      // cannot yield a row (:291), but keeps its rank
        candidate_modes(   // over the whole hit list, filtered by id
            a, sh.ms, hist, filt, qi, nhits,
            [&](int i, int& d) { const uint2 h = hits[i]; d = (int)h.y; return h.x == bid; }, bid, raw, rank);
      }
    }
    __syncthreads();
    if (tid == 0) query_done(a, qi, sh.ms.nrows, maxdepth, nabove);
    __syncthreads();
  }
}

// ---- get_hits (hash_table.py:150-176) -----------------------------------------
__global__ void afp_hit_count_kernel(const int32_t* q, int64_t nq, const int32_t* counts, int hashbits,
                                     int depth, int32_t* n_out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq) return;
  const uint32_t b = (uint32_t)q[2 * i + 1] & ((1u << hashbits) - 1u);
  n_out[i] = min(depth, counts[b]);
}

__global__ void afp_hit_write_kernel(const int32_t* q, int64_t nq, const uint32_t* table, const int32_t* counts,
                                     int hashbits, int depth, int mtb, const int64_t* off, int32_t* hits) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  if (r >= nq) return;
  const int lane = threadIdx.x & 31;
  const int qt = q[2 * r];
  const uint32_t b = (uint32_t)q[2 * r + 1] & ((1u << hashbits) - 1u);
  const int n = min(depth, counts[b]);
  const uint32_t tmask = (1u << mtb) - 1u;
  const uint32_t* row = table + (size_t)b * depth;
  int32_t* out = hits + 4 * off[r];
  for (int s = lane; s < n; s += 32) {
    const uint32_t v = row[s];
    out[4 * s + 0] = (int32_t)((v >> mtb) - 1u);
    out[4 * s + 1] = (int32_t)(v & tmask) - qt;
    out[4 * s + 2] = (int32_t)b;
    out[4 * s + 3] = qt;
  }
}

__global__ void afp_restrict_ids_kernel(uint32_t* table, int32_t* counts, int64_t nbuckets, int depth, int mtb,
                                        uint32_t id_lo, uint32_t id_hi) {
  const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nbuckets) return;
  uint32_t* row = table + (size_t)b * depth;
  const int n = min(depth, counts[b]);
  int k = 0;
  for (int s = 0; s < n; ++s) {
    const uint32_t v = row[s];
    const uint32_t id = (v >> mtb) - 1u;
    if (id >= id_lo && id < id_hi) row[k++] = v;
  }
  for (int s = k; s < n; ++s) row[s] = 0;
  counts[b] = k;
}

// smallest non-zero hashesperid and the number of zero entries (tracks removed, or never filled)
__global__ void afp_hpi_stats_kernel(const uint32_t* hpi, int64_t nids, unsigned* out /* [min, nzero] */) {
  unsigned mn = 0xffffffffu, nz = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nids; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned h = hpi[i];
    if (h) mn = min(mn, h); else ++nz;
  }
  mn = __reduce_min_sync(0xffffffffu, mn);
  nz = __reduce_add_sync(0xffffffffu, nz);
  if ((threadIdx.x & 31) == 0) { atomicMin(&out[0], mn); if (nz) atomicAdd(&out[1], nz); }
}
// does any live table entry name a track whose hashesperid is zero?  (Then a weight can be
// infinite and the fast path's pruning bound does not hold: it runs without pruning.)
__global__ void afp_refzero_kernel(const uint32_t* table, const int32_t* counts, int64_t nbuckets, int depth, int mtb,
                                   const uint32_t* hpi, int64_t nids, unsigned* flag) {
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= nbuckets) return;
  const int n = min(depth, counts[b]);
  bool bad = false;
  for (int s = threadIdx.x & 31; s < n; s += 32) {
    const uint32_t id = (table[(size_t)b * depth + s] >> mtb) - 1u;
    if (id < (uint32_t)nids && hpi[id] == 0u) bad = true;
  }
  if (bad) atomicExch(flag, 1u);
}

__global__ void afp_qmax_kernel(const int32_t* q, int64_t nq, int* out_max, int* out_min) {
  int mx = 0, mn = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nq; i += (int64_t)gridDim.x * blockDim.x) {
    mx = max(mx, q[2 * i]);
    mn = min(mn, q[2 * i]);
  }
  mx = __reduce_max_sync(0xffffffffu, mx);
  mn = __reduce_min_sync(0xffffffffu, mn);
  if ((threadIdx.x & 31) == 0) { atomicMax(out_max, mx); atomicMin(out_min, mn); }
}

__global__ void afp_pack_rows_kernel(const int32_t* rows, const int32_t* row_cnt, const int64_t* off, int row_cap,
                                     int32_t* packed) {
  const int qi = blockIdx.x;
  const int n = min(row_cnt[qi], row_cap);
  const int32_t* src = rows + (size_t)qi * row_cap * 7;
  int32_t* dst = packed + 7 * off[qi];
  for (int i = threadIdx.x; i < n * 7; i += blockDim.x) dst[i] = src[i];
}

__global__ void afp_clamp_kernel(const int32_t* in, int n, int cap, int32_t* out, int* overflow) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (in[i] > cap) atomicExch(overflow, 1);
  out[i] = min(in[i], cap);
}

}  // namespace

// Rows of a batch sit at a fixed stride (row_cap per query) in d_mrows with their counts in
// d_mrow_cnt: clamp the counts to the capacity (flagging overflow), scan, pack -> d_mrows_packed,
// d_mrow_off (what afp_fetch_match_rows returns).
int afp_finish_match_rows(afp_ctx* c, int nqueries, int row_cap, int64_t* total_out) {
  int* d_over = c->d_mrow_cnt.as<int>() + nqueries + 1;
  AFP_CUDA(c, cudaMemsetAsync(d_over, 0, sizeof(int), c->stream));
  AFP_CUDA(c, c->d_tmp.reserve(sizeof(int32_t) * (size_t)(nqueries + 8)));
  int64_t total = 0;
  int over = 0;
  int rc;
  if ((rc = afp_launch(c, afp_clamp_kernel, (nqueries + 255) / 256, 256, 0, c->d_mrow_cnt.as<int32_t>(), nqueries,
                       row_cap, c->d_tmp.as<int32_t>(), d_over)) ||
      (rc = afp_launch_scan_i32_to_i64(c, c->d_tmp.as<int32_t>(), c->d_mrow_off.as<int64_t>(), nqueries)) ||
      (rc = afp_read_back(c, &total, c->d_mrow_off.as<int64_t>() + nqueries, 1, &over, d_over, 1)))
    return rc;
  if (over) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "row capacity exceeded: a query produced more rows than afp_matcher_params.row_capacity");
  AFP_CUDA(c, c->d_mrows_packed.reserve(sizeof(int32_t) * 7 * (size_t)(total + 1)));
  if (total > 0 &&
      (rc = afp_launch(c, afp_pack_rows_kernel, nqueries, 64, 0, c->d_mrows.as<int32_t>(), c->d_mrow_cnt.as<int32_t>(),
                       c->d_mrow_off.as<int64_t>(), row_cap, c->d_mrows_packed.as<int32_t>())))
    return rc;
  c->match_total_rows = total;
  *total_out = total;
  return AFP_OK;
}

extern "C" {

int afp_table_upload(afp_ctx* c, const uint32_t* table, const int32_t* counts, int32_t hashbits, int32_t depth,
                     int32_t maxtimebits, const uint32_t* hashesperid, int64_t nids, int on_host) {
  if (!c || !table || !counts || (nids > 0 && !hashesperid)) return AFP_ERR_INVALID;
  if (hashbits < 1 || hashbits > 28 || depth < 1 || maxtimebits < 1 || maxtimebits > 24 || nids < 0)
    AFP_FAIL(c, AFP_ERR_INVALID, "bad table geometry");
  AFP_CUDA(c, cudaSetDevice(c->device));
  const size_t nb = (size_t)1 << hashbits;
  c->tab.loaded = false;
  AFP_CUDA(c, c->tab.table.reserve(nb * (size_t)depth * sizeof(uint32_t)));
  AFP_CUDA(c, c->tab.counts.reserve(nb * sizeof(int32_t)));
  AFP_CUDA(c, c->tab.hashesperid.reserve(((size_t)nids + 1) * sizeof(uint32_t)));
  AFP_CUDA(c, afp_copy_in(c, c->tab.table.as<uint32_t>(), table, nb * (size_t)depth, on_host));
  AFP_CUDA(c, afp_copy_in(c, c->tab.counts.as<int32_t>(), counts, nb, on_host));
  if (nids > 0) AFP_CUDA(c, afp_copy_in(c, c->tab.hashesperid.as<uint32_t>(), hashesperid, (size_t)nids, on_host));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  c->tab.hashbits = hashbits;
  c->tab.depth = depth;
  c->tab.maxtimebits = maxtimebits;
  c->tab.nids = nids;
  c->tab.loaded = true;
  return afp_table_stats(c);
}

// min(hashesperid) for the fast matching path's pruning bound (0 = do not prune)
int afp_table_stats(afp_ctx* c) {
  c->tab.hmin = 0;
  if (c->tab.nids <= 0) return AFP_OK;
  AFP_CUDA(c, c->d_tmp.reserve(64));
  unsigned* d = c->d_tmp.as<unsigned>();
  const unsigned init[3] = {0xffffffffu, 0u, 0u};
  AFP_CUDA(c, cudaMemcpyAsync(d, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
  unsigned h[3];
  int rc;
  if ((rc = afp_launch(c, afp_hpi_stats_kernel, 296, 256, 0, c->tab.hashesperid.as<uint32_t>(), c->tab.nids, d)) ||
      (rc = afp_read_back(c, h, d, 3)))
    return rc;
  if (h[1] != 0u) {          // zero entries exist: harmless as long as no table entry names them
    const int64_t nb = (int64_t)1 << c->tab.hashbits;
    if ((rc = afp_launch(c, afp_refzero_kernel, (unsigned)((nb + 7) / 8), 256, 0, c->tab.table.as<uint32_t>(),
                         c->tab.counts.as<int32_t>(), nb, c->tab.depth, c->tab.maxtimebits,
                         c->tab.hashesperid.as<uint32_t>(), c->tab.nids, d + 2)) ||
        (rc = afp_read_back(c, h, d, 3)))
      return rc;
  }
  c->tab.hmin = (h[0] != 0xffffffffu && h[2] == 0u) ? h[0] : 0u;
  return AFP_OK;
}

int afp_table_pruning_bound(afp_ctx* c, uint32_t* hmin) {
  if (!c || !hmin) return AFP_ERR_INVALID;
  if (!c->tab.loaded) AFP_FAIL(c, AFP_ERR_STATE, "no table on the device");
  *hmin = c->tab.hmin;
  return AFP_OK;
}

int afp_table_restrict_ids(afp_ctx* c, int64_t id_lo, int64_t id_hi) {
  if (!c) return AFP_ERR_INVALID;
  if (!c->tab.loaded) AFP_FAIL(c, AFP_ERR_STATE, "no table uploaded");
  if (id_lo < 0 || id_hi < id_lo) AFP_FAIL(c, AFP_ERR_INVALID, "bad id range");
  AFP_CUDA(c, cudaSetDevice(c->device));
  const int64_t nb = (int64_t)1 << c->tab.hashbits;
  return afp_launch(c, afp_restrict_ids_kernel, (unsigned)((nb + 255) / 256), 256, 0, c->tab.table.as<uint32_t>(),
                    c->tab.counts.as<int32_t>(), nb, c->tab.depth, c->tab.maxtimebits, (uint32_t)id_lo,
                    (uint32_t)id_hi);
}

int afp_get_hits(afp_ctx* c, const int32_t* q_rows, int64_t nq, int q_on_host, int64_t* nhits) {
  if (!c || nq < 0 || (nq > 0 && !q_rows)) return AFP_ERR_INVALID;
  if (!c->tab.loaded) AFP_FAIL(c, AFP_ERR_STATE, "no table uploaded");
  AFP_CUDA(c, cudaSetDevice(c->device));
  c->nhits = -1;
  const int32_t* dq = nullptr;
  int rc = afp_stage(c, c->d_q, q_rows, 2 * (size_t)nq, q_on_host, &dq);
  if (rc) return rc;
  AFP_CUDA(c, c->d_tmp.reserve(sizeof(int32_t) * (size_t)(nq + 1)));
  AFP_CUDA(c, c->d_hit_off.reserve(sizeof(int64_t) * (size_t)(nq + 1)));
  int64_t total = 0;
  if ((rc = afp_launch(c, afp_hit_count_kernel, (unsigned)((nq + 255) / 256), 256, 0, dq, nq,
                       c->tab.counts.as<int32_t>(), c->tab.hashbits, c->tab.depth, c->d_tmp.as<int32_t>())) ||
      (rc = afp_launch_scan_i32_to_i64(c, c->d_tmp.as<int32_t>(), c->d_hit_off.as<int64_t>(), nq)) ||
      (rc = afp_read_back(c, &total, c->d_hit_off.as<int64_t>() + nq, 1)))
    return rc;
  AFP_CUDA(c, c->d_hits.reserve(sizeof(int32_t) * 4 * (size_t)(total + 1)));
  if (total > 0 &&
      (rc = afp_launch(c, afp_hit_write_kernel, (unsigned)((nq + 7) / 8), 256, 0, dq, nq, c->tab.table.as<uint32_t>(),
                       c->tab.counts.as<int32_t>(), c->tab.hashbits, c->tab.depth, c->tab.maxtimebits,
                       c->d_hit_off.as<int64_t>(), c->d_hits.as<int32_t>())))
    return rc;
  c->nhits = total;
  c->hits_nq = nq;
  if (nhits) *nhits = total;
  return AFP_OK;
}

int afp_fetch_hits(afp_ctx* c, int32_t* hits, int hits_on_host) {
  if (!c) return AFP_ERR_INVALID;
  if (c->nhits < 0) AFP_FAIL(c, AFP_ERR_STATE, "afp_get_hits has not been called");
  AFP_CUDA(c, cudaSetDevice(c->device));
  if (hits && c->nhits > 0) AFP_CUDA(c, afp_copy_out(c, hits, c->d_hits.as<int32_t>(), 4 * (size_t)c->nhits, hits_on_host));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  return AFP_OK;
}

int afp_match_batch(afp_ctx* c, const int32_t* q_rows, int q_on_host, int32_t nqueries, const int64_t* q_offsets,
                    const afp_matcher_params* p, int64_t* total_rows) {
  if (!c || !p || nqueries < 0 || (nqueries > 0 && !q_offsets)) return AFP_ERR_INVALID;
  if (!c->tab.loaded) AFP_FAIL(c, AFP_ERR_STATE, "no table uploaded");
  if (p->window < 0 || p->window > 4096 || p->threshcount < 0 || p->search_depth < 0 || p->max_alignments_per_id < 0)
    AFP_FAIL(c, AFP_ERR_INVALID, "bad matcher parameters");
  AFP_CUDA(c, cudaSetDevice(c->device));
  c->match_total_rows = -1;
  c->match_nq = nqueries;
  c->match_long.clear();
  c->sopt.pending = c->sopt.finished = false;
  // A query of rows * depth >= AFP_LONG_HITS takes the long-query path (afp_match_long.cu) unless
  // force_general is set; the rule depends on the query and the table only.  The fast and general
  // kernels' scratch is sized over the other queries.
  int64_t maxnq = 0;
  std::vector<int> longq;
  for (int i = 0; i < nqueries; ++i) {
    if (q_offsets[i + 1] < q_offsets[i]) AFP_FAIL(c, AFP_ERR_INVALID, "q_offsets must be non-decreasing");
    const int64_t n = q_offsets[i + 1] - q_offsets[i];
    if (!p->force_general && n * c->tab.depth >= AFP_LONG_HITS) {
      if (n >= ((int64_t)1 << 31)) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "query of 2^31 rows or more");
      longq.push_back(i);
    } else {
      maxnq = std::max<int64_t>(maxnq, n);
    }
  }
  const int nlong = (int)longq.size(), nshort = nqueries - nlong;
  const int64_t nrows_in = nqueries ? q_offsets[nqueries] : 0;
  if (nqueries && q_offsets[0] != 0) AFP_FAIL(c, AFP_ERR_INVALID, "q_offsets[0] must be 0");
  if (nrows_in > 0 && !q_rows) return AFP_ERR_INVALID;
  const int32_t* dq = nullptr;
  int rc = afp_stage(c, c->d_q, q_rows, 2 * (size_t)nrows_in, q_on_host, &dq);
  if (rc) return rc;
  AFP_CUDA(c, c->d_qoff.reserve(sizeof(int64_t) * (size_t)(nqueries + 1)));
  AFP_CUDA(c, c->d_mrow_cnt.reserve(sizeof(int32_t) * (size_t)(nqueries + 2)));
  AFP_CUDA(c, c->d_mrow_off.reserve(sizeof(int64_t) * (size_t)(nqueries + 1)));
  if (nqueries == 0) {
    c->match_total_rows = 0;
    if (total_rows) *total_rows = 0;
    return AFP_OK;
  }
  AFP_CUDA(c, cudaMemcpyAsync(c->d_qoff.p, q_offsets, sizeof(int64_t) * (size_t)(nqueries + 1),
                              cudaMemcpyHostToDevice, c->stream));
  // largest / smallest query time (sizes the dtime histogram): [0, 1] over the fast / general
  // kernels' queries, [2, 3] over the long ones (the row ranges in between are contiguous)
  int h_mm[4] = {0, 0, 0, 0};
  AFP_CUDA(c, c->d_tmp.reserve(sizeof(int32_t) * (size_t)(nqueries + 8)));
  int* d_mm = c->d_tmp.as<int>();
  AFP_CUDA(c, cudaMemsetAsync(d_mm, 0, 4 * sizeof(int), c->stream));
  auto qmax = [&](int64_t r0, int64_t r1, int* out) {
    return r1 <= r0 ? AFP_OK : afp_launch(c, afp_qmax_kernel, 296, 256, 0, dq + 2 * r0, r1 - r0, out, out + 1);
  };
  {
    int64_t r0 = 0;
    for (int li : longq) {
      if ((rc = qmax(r0, q_offsets[li], d_mm)) || (rc = qmax(q_offsets[li], q_offsets[li + 1], d_mm + 2))) return rc;
      r0 = q_offsets[li + 1];
    }
    if ((rc = qmax(r0, nrows_in, d_mm)) || (rc = afp_read_back(c, h_mm, d_mm, 4))) return rc;
  }
  if (h_mm[1] < 0 || h_mm[3] < 0) AFP_FAIL(c, AFP_ERR_INVALID, "negative query time");
  // dtime histogram: bin dt + bias for dt in [-qmax, 2^maxtimebits), bias = qmax + window + 2,
  // indexed with int by the kernels.  [0] short queries, [1] long ones.
  int64_t bias[2], hist_len[2];
  for (int k = 0; k < 2; ++k) {
    bias[k] = (int64_t)h_mm[2 * k] + p->window + 2;
    hist_len[k] = ((int64_t)1 << c->tab.maxtimebits) + bias[k] + p->window + 4;
    if (hist_len[k] > INT32_MAX)
      AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "query time too large: 2^maxtimebits + query time + 2 * window + 6 must not exceed 2^31 - 1");
  }

  // persistent grid; a fixed CTA count keeps the scratch layout (and its zeroed state) reusable
  int nctas = c->num_sms;
  MatchArgs a;
  a.q = dq;
  a.qoff = c->d_qoff.as<int64_t>();
  a.nqueries = nqueries;
  a.table = c->tab.table.as<uint32_t>();
  a.counts = c->tab.counts.as<int32_t>();
  a.hpi = c->tab.hashesperid.as<uint32_t>();
  a.hashbits = c->tab.hashbits;
  a.depth = c->tab.depth;
  a.mtb = c->tab.maxtimebits;
  a.nids = std::max<int64_t>(c->tab.nids, 1);
  a.window = p->window;
  a.thresh = p->threshcount;
  a.sdepth = p->search_depth;
  a.maxalign = p->max_alignments_per_id;
  a.hits_cap = std::max<int64_t>(maxnq * c->tab.depth, 1);
  a.bias = (int)bias[0];
  a.hist_len = (int)hist_len[0];
  a.row_cap = p->row_capacity > 0 ? p->row_capacity : 256;
  if (a.hits_cap >= HITS_MAX || a.nids >= ((int64_t)1 << 24))
    AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "query too large (rows * depth >= 2^30) or more than 2^24 track ids");
  const size_t per_cta = (size_t)a.hits_cap * (sizeof(uint2) + 4 * sizeof(uint32_t) + sizeof(double)) +
                         (size_t)a.hist_len * 2 * sizeof(int32_t) + 256;
  // The scratch is per CTA and sized for the longest query the fast / general kernels run (whole
  // shows, searching_for_ads.md, take the long-query path): when it would not fit the memory
  // budget the grid shrinks instead of the call failing.
  size_t budget = 0;
  AFP_CUDA(c, afp_memory_budget(c->d_mscratch, &budget));
  if (per_cta * (size_t)nctas > budget) nctas = (int)std::max<size_t>(1, budget / per_cta);
  if (per_cta > budget) AFP_FAIL(c, AFP_ERR_NOMEM, "match scratch of one query exceeds the device memory budget");
  const size_t before = c->d_mscratch.cap;
  AFP_CUDA(c, c->d_mrows.reserve(sizeof(int32_t) * 7 * (size_t)a.row_cap * (size_t)nqueries));
  // carve the scratch; the histograms at its end must start (and are left) zeroed
  const int64_t per_hit = a.hits_cap * nctas, per_bin = (int64_t)a.hist_len * nctas;
  size_t zero0 = 0, zero1 = 0;
  if ((rc = afp_carve(c, c->d_mscratch, [&](Carver& k) {
         a.hits = k.take<uint2>(per_hit);
         a.wtd = k.take<double>(per_hit);
         a.dlist = k.take<uint32_t>(per_hit);
         a.dts = k.take<uint32_t>(per_hit);
         a.recs = k.take<uint32_t>(per_hit);
         a.rawl = k.take<uint32_t>(per_hit);
         zero0 = k.bytes;
         a.hist = k.take<int32_t>(per_bin);
         a.filt = k.take<int32_t>(per_bin);
         zero1 = k.bytes;
       })))
    return rc;
  // the histograms are left zeroed by the kernel itself: clear them only when the
  // carve-up changed (or the buffer moved)
  const uint64_t layout = (uint64_t)a.hits_cap * 1000003ull ^ (uint64_t)a.nids * 7919ull ^ (uint64_t)a.hist_len * 31ull ^
                          (uint64_t)(uintptr_t)c->d_mscratch.p ^ (uint64_t)before ^ (uint64_t)nctas * 2654435761ull;
  if (layout != c->match_layout) {
    AFP_CUDA(c, cudaMemsetAsync(c->d_mscratch.as<char>() + zero0, 0, zero1 - zero0, c->stream));
    c->match_layout = layout;
  }
  a.rows = c->d_mrows.as<int32_t>();
  a.row_cnt = c->d_mrow_cnt.as<int32_t>();
  a.publish = p->publish_candidates ? 1 : 0;
  a.cand = nullptr;
  a.cand_cnt = nullptr;
  c->match_published = false;
  if (a.publish) {
    AFP_CUDA(c, c->d_mcand.reserve(sizeof(double) * 3 * (size_t)std::max(a.sdepth, 1) * (size_t)nqueries));
    AFP_CUDA(c, c->d_mcand_cnt.reserve(sizeof(int32_t) * 2 * (size_t)nqueries));
    a.cand = c->d_mcand.as<double>();
    a.cand_cnt = c->d_mcand_cnt.as<int32_t>();
    c->match_sdepth = a.sdepth;
    c->match_published = true;
  }
  c->match_row_cap = a.row_cap;
  // ---- fast path first (afp_match_fast.cu); whatever it cannot take goes to the general kernel
  a.qlist = nullptr;
  a.nlist = nullptr;
  a.fstat = nullptr;
  a.qskip = nullptr;
  c->match_fast_ran = false;
  a.mhits = nullptr;
  a.mh_cap = 0;
  a.hmin = c->tab.hmin;
  a.bm_exact = c->tab.nids <= ((int64_t)1 << 20) ? 1 : 0;
  const bool fast = !p->force_general && p->threshcount >= 1 && p->search_depth >= 1 && c->tab.depth <= 65535 &&
                    a.hist_len < (1 << 30);
  c->match_general = nshort;
  if (fast || nlong) {
    // [count + pad][query list][status: 8 per query][long-query flags, bytes]
    AFP_CUDA(c, c->d_mqlist.reserve(sizeof(int32_t) * (size_t)(9 * nqueries + 4) + (size_t)nqueries));
    a.nlist = c->d_mqlist.as<int>();
    a.qlist = c->d_mqlist.as<int32_t>() + 4;
    a.fstat = a.qlist + nqueries;
  }
  std::vector<int32_t> h_list;
  std::vector<unsigned char> h_skip;
  if (nlong) {
    // the fast kernel skips the long queries; without it, the general kernel gets the others as its list
    h_skip.assign(nqueries, 0);
    for (int li : longq) h_skip[li] = 1;
    unsigned char* d_skip = reinterpret_cast<unsigned char*>(a.fstat + 8 * (size_t)nqueries);
    AFP_CUDA(c, cudaMemcpyAsync(d_skip, h_skip.data(), (size_t)nqueries, cudaMemcpyHostToDevice, c->stream));
    a.qskip = d_skip;
    if (!fast) {
      h_list.assign(1, nshort);
      h_list.resize(4, 0);
      for (int i = 0; i < nqueries; ++i)
        if (!h_skip[i]) h_list.push_back(i);
      AFP_CUDA(c, cudaMemcpyAsync(a.nlist, h_list.data(), sizeof(int32_t) * h_list.size(), cudaMemcpyHostToDevice,
                                  c->stream));
    }
  } else if (!fast) {
    a.qlist = nullptr;
    a.nlist = nullptr;
    a.fstat = nullptr;
  }
  if (fast && nshort) {
    a.mh_cap = (int)std::min<int64_t>(std::max<int64_t>((a.hits_cap + 31) / 32 * 32, 32768), 131072);   // 32 per-warp segments
    AFP_CUDA(c, c->d_mfast.reserve(sizeof(uint2) * (size_t)a.mh_cap * (size_t)nctas));
    a.mhits = c->d_mfast.as<uint2>();
    AFP_CUDA(c, cudaMemsetAsync(a.nlist, 0, sizeof(int), c->stream));
    if ((rc = afp_launch_match_fast(c, a, nctas))) return rc;
    c->match_fast_ran = true;
  }
  if (nshort && (rc = afp_launch(c, afp_match_kernel, nctas, MT, QCAP * sizeof(unsigned long long), a))) return rc;
  if (c->match_fast_ran) AFP_CUDA(c, afp_read_async(c, &c->match_general_h, a.nlist, 1));
  if (nlong) {
    // ---- long queries (afp_match_long.cu): one histogram pair per CTA of the mode pass, sized
    // over the long queries' times, zeroed here and left zeroed by the mode search
    MatchArgs al = a;
    al.bias = (int)bias[1];
    al.hist_len = (int)hist_len[1];
    const size_t per = (size_t)al.hist_len * 2 * sizeof(int32_t);
    AFP_CUDA(c, afp_memory_budget(c->d_lg_hist, &budget));
    c->lg_ctas = (int)std::max<size_t>(1, std::min<size_t>((size_t)c->num_sms, budget / per));
    AFP_CUDA(c, c->d_lg_hist.reserve(per * (size_t)c->lg_ctas));
    al.hist = c->d_lg_hist.as<int32_t>();
    al.filt = al.hist + (size_t)al.hist_len * c->lg_ctas;
    AFP_CUDA(c, cudaMemsetAsync(al.hist, 0, sizeof(int32_t) * (size_t)al.hist_len * c->lg_ctas, c->stream));
    for (int li : longq)
      if ((rc = afp_match_long(c, al, li, q_offsets[li], q_offsets[li + 1] - q_offsets[li]))) return rc;
    c->match_long = longq;
  }
  int64_t total = 0;
  if ((rc = afp_finish_match_rows(c, nqueries, a.row_cap, &total))) return rc;
  if (c->match_fast_ran) c->match_general = c->match_general_h;     // (the stream was synchronised)
  if (total_rows) *total_rows = total;
  return AFP_OK;
}

int afp_match_general_count(afp_ctx* c, int64_t* n) {
  if (!c || !n) return AFP_ERR_INVALID;
  if (c->match_total_rows < 0) AFP_FAIL(c, AFP_ERR_STATE, "afp_match_batch has not been called");
  *n = c->match_general;
  return AFP_OK;
}

int afp_fetch_match_status(afp_ctx* c, int32_t* status) {
  if (!c || !status) return AFP_ERR_INVALID;
  if (c->match_total_rows < 0) AFP_FAIL(c, AFP_ERR_STATE, "afp_match_batch has not been called");
  AFP_CUDA(c, cudaSetDevice(c->device));
  if (!c->match_fast_ran) {
    for (int i = 0; i < 8 * c->match_nq; ++i) status[i] = -1;
  } else {
    const int rc = afp_read_back(c, status, c->d_mqlist.as<int32_t>() + 4 + c->match_nq, 8 * (size_t)c->match_nq);
    if (rc) return rc;
  }
  for (int qi : c->match_long) {          // finished by the long-query path
    status[8 * (size_t)qi] = 6;
    for (int k = 1; k < 8; ++k) status[8 * (size_t)qi + k] = 0;
  }
  return AFP_OK;
}

int afp_fetch_match_candidates(afp_ctx* c, double* cand, int32_t* counts, int on_host) {
  if (!c) return AFP_ERR_INVALID;
  if (c->match_total_rows < 0 || !c->match_published)
    AFP_FAIL(c, AFP_ERR_STATE, "afp_match_batch with publish_candidates has not been called");
  AFP_CUDA(c, cudaSetDevice(c->device));
  if (cand && c->match_nq > 0 && c->match_sdepth > 0)
    AFP_CUDA(c, afp_copy_out(c, cand, c->d_mcand.as<double>(), 3 * (size_t)c->match_sdepth * (size_t)c->match_nq,
                             on_host));
  if (counts && c->match_nq > 0)
    AFP_CUDA(c, afp_copy_out(c, counts, c->d_mcand_cnt.as<int32_t>(), 2 * (size_t)c->match_nq, on_host));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  return AFP_OK;
}

int afp_fetch_match_rows(afp_ctx* c, int32_t* rows, int rows_on_host, int64_t* row_offsets) {
  if (!c) return AFP_ERR_INVALID;
  if (c->match_total_rows < 0) AFP_FAIL(c, AFP_ERR_STATE, "afp_match_batch has not been called");
  AFP_CUDA(c, cudaSetDevice(c->device));
  if (row_offsets) {
    if (c->match_nq == 0) row_offsets[0] = 0;
    else AFP_CUDA(c, afp_copy_out(c, row_offsets, c->d_mrow_off.as<int64_t>(), (size_t)(c->match_nq + 1), 1));
  }
  if (rows && c->match_total_rows > 0)
    AFP_CUDA(c, afp_copy_out(c, rows, c->d_mrows_packed.as<int32_t>(), 7 * (size_t)c->match_total_rows, rows_on_host));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  return AFP_OK;
}

}  // extern "C"
