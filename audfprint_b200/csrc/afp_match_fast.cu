// K4 fast path — probe + exact candidate ranking without materialising the hit list.
//
// Same results as the general kernel (afp_match.cu), i.e. HashTable.get_hits
// (hash_table.py:150-176) -> Matcher._best_count_ids (audfprint_match.py:124-147) ->
// Matcher._approx_match_counts (:241-312), for the common case: threshcount >= 1, candidate depth
// <= 1024, a few thousand track ids hit more than once.  Queries outside its capacities are
// handed to the general kernel through a work list, so the pair is exact for every input.
//
// Why it is faster (the general kernel spends ~4 shared-memory atomics + ~90 bytes of HBM scratch
// per probed table entry): a 10 s query touches ~80k table entries but only a few thousand track ids
// more than once, and only those can matter -
//   * an id hit by ONE (bucket, slot) record has raw count m = the number of query rows that
//     probe that bucket (<= shifts, and <= threshcount or it is treated as a multi-record id), so
//     it can never produce a result row (needs a dtime bin > threshcount) and can reach the
//     candidate list only through its weight m / hashesperid[id];
//   * pass 1 therefore only finds the multi-record ids: ONE shared-memory atomicOr per entry on
//     a 2^20-bit "seen" bitmap; an entry whose bit was already set puts its id into a small
//     open-addressing set (a hashed bitmap for > 2^20 ids only adds false members, which are
//     then counted exactly like any other member);
//   * pass 2 re-reads the same bucket rows (L2 hits: the CTA read them microseconds ago),
//     tests every entry against a "member" bitmap (one shared-memory load) and appends the hits
//     (set slot, dtime) of members to a short list; the exact raw counts are then a histogram
//     of that list;
//   * the top-K members by (weight desc, id desc) come from a histogram select on the float
//     image of the weight (monotone), then a bitonic sort of the few hundred survivors (cheaper than
//     a full sort of the ~6000 members);
//     single-record ids are provably out when  min(m_max, threshcount) / min(hashesperid) <
//     K-th member weight; otherwise pass 3 re-reads only the bucket groups whose multiplicity
//     could reach that weight, gathers hashesperid for their non-member ids and admits the
//     few that do outrank the K-th member;
//   * the hits of the row-capable candidates are routed from the member list; the candidate stage
//     around that routing (dt-list offsets, quick filter, histogram mode search) is the general
//     kernel's, from afp_match_common.cuh.
// Per probed entry: 4 B read from HBM, 4 B again from L2, one atomicOr, one set lookup.
#include "afp_match_common.cuh"

namespace {

constexpr int BM_BITS = 1 << 20;            // "seen" / "member" bitmaps, one bit per (hashed) track id: 128 KB
constexpr int BM_WORDS = BM_BITS / 32;
constexpr int MSLOTS = 16384;               // open-addressing set of multi-record ids (keys: 64 KB)
constexpr int MMAX = 12288;                 // members the set may hold (load factor <= 0.75)
constexpr int QF = 2048;                    // query rows sorted per chunk
constexpr int SCAP = 4096;                  // rank-sort capacity: selected members + admitted single-record ids
constexpr int XCAP = 2048;                  // single-record ids pass 3 may admit
constexpr int PROBE_MAX = 256;              // insertion gives up (set full) after this many probes
constexpr int WBINS = 4096;                 // weight histogram bins (float image of the weight, top 16 bits)
// why a query was handed to the general kernel (afp_fetch_match_status)
enum { FS_DONE = 0, FS_SET_FULL = 1, FS_HITS_FULL = 2, FS_EXTRAS_FULL = 3, FS_NDIST_UNKNOWN = 4, FS_DEPTH = 5,
       FS_INCONSISTENT = 6, FS_TIES = 7 };

// dynamic shared memory (bytes).  R0 is the "seen" bitmap in pass 1, the "member" bitmap in
// pass 2, then the member counters + selection / rank arrays; R2 holds the sorted query chunk
// and its bucket groups during the passes and the slot -> candidate map afterwards.
constexpr int OFF_R0 = 0;                                  // u32 bitmap[BM_WORDS]
constexpr int OFF_MCNT = OFF_R0;                           //   u32 mcnt[MSLOTS]            (after pass 2)
constexpr int OFF_WH = OFF_R0 + MSLOTS * 4;                //   int whist[WBINS]            (selection)
constexpr int OFF_SW = OFF_R0 + MSLOTS * 4;                //   u64 sw[SCAP]                (ranking; over whist)
constexpr int OFF_SID = OFF_SW + SCAP * 8;                 //   u32 sid[SCAP]
constexpr int OFF_SRAW = OFF_SID + SCAP * 4;               //   u32 sraw[SCAP]
constexpr int OFF_MKEYS = OFF_R0 + BM_WORDS * 4;           // u32 mkeys[MSLOTS] (id + 1, 0 = empty)
constexpr int OFF_Q = OFF_MKEYS + MSLOTS * 4;              // u64 qkeys[QF]
constexpr int OFF_HPOS = OFF_Q + QF * 8;                   // u16 hpos[QF], hm[QF], hn[QF]
constexpr int GBINS = 1024;                                //   int gbin[GBINS]: counting sort of the chunk
constexpr int OFF_GBIN = OFF_HPOS + QF * 6;
constexpr int OFF_MAP = OFF_Q;                             //   u16 map16[MSLOTS]           (routing)
constexpr int FAST_SMEM = OFF_HPOS + QF * 8;               // 229376 B
static_assert(OFF_SRAW + SCAP * 4 == OFF_MKEYS, "rank arrays fill the upper half of R0");
static_assert(WBINS * 4 <= SCAP * 8, "weight histogram fits under sw");
static_assert(MSLOTS * 2 <= QF * 16, "slot map fits R2");
static_assert(OFF_GBIN + GBINS * 4 <= OFF_HPOS + QF * 8, "bin counters fit behind the group arrays");
// after the final sort only the first KCAP ranks are alive: the dt-list bookkeeping of the
// candidates reuses the tail of sid[]
constexpr int OFF_LOFF = OFF_SID + KCAP * 4;
constexpr int OFF_CUR = OFF_LOFF + KCAP * 4;
constexpr int OFF_PASS = OFF_CUR + KCAP * 4;
static_assert(OFF_PASS + KCAP <= OFF_SRAW, "candidate bookkeeping fits behind sid[0..KCAP)");

struct FastShared {
  ModeScratch ms;
  int wsum[NW];
  int wcount[NW];          // hits in every warp's segment of the member-hit list
  unsigned nmem, nmh, nx, nabove, ndist, mmax, ngath;
  int overflow;
  int cut_bin, cut_above;
};

__device__ __forceinline__ unsigned bm_index(unsigned id, int exact) {
  return exact ? id : (id * 2654435761u) >> 12;
}
__device__ __forceinline__ unsigned set_hash(unsigned id) { return (id * 0x9E3779B1u) >> 18; }   // 14 bits

// slot of `id` in the member set, -1 if absent (the set is not modified concurrently)
__device__ __forceinline__ int set_find(const unsigned* mkeys, unsigned id) {
  const unsigned key = id + 1u;
  unsigned h = set_hash(id);
  while (true) {
    const unsigned k = mkeys[h];
    if (k == key) return (int)h;
    if (k == 0u) return -1;
    h = (h + 1u) & (MSLOTS - 1);
  }
}

// histogram bin of a weight: the top 16 bits of its float image (8 exponent + 7 mantissa bits),
// rebased so that 2^-24 .. 2^8 covers WBINS bins; monotone non-decreasing in the weight
__device__ __forceinline__ int weight_bin(double w) {
  const int b = (int)(__float_as_uint((float)w) >> 16) - (((127 - 24) << 7));
  return min(max(b, 0), WBINS - 1);
}

// Sort one chunk of query rows by (bucket, time) and list its bucket groups:
// hpos[g] = first row of group g, hm[g] = rows probing that bucket, hn[g] = slots to read.
__device__ int prepare_chunk(const MatchArgs& a, FastShared& fs, unsigned char* smem, int64_t row0, int n) {
  unsigned long long* qkeys = reinterpret_cast<unsigned long long*>(smem + OFF_Q);
  unsigned short* hpos = reinterpret_cast<unsigned short*>(smem + OFF_HPOS);
  unsigned short* hm = hpos + QF;
  unsigned short* hn = hm + QF;
  const int tid = threadIdx.x;
  const uint32_t hmask = (1u << a.hashbits) - 1u;
  // Group the rows by bucket without a full sort: counting sort into GBINS hash bins of the
  // bucket (two shared-memory atomics per row), then every bin's handful of keys is put in
  // order by one thread.  Equal buckets end up adjacent, their times ascending.
  int* gbin = reinterpret_cast<int*>(smem + OFF_GBIN);
  static_assert(GBINS == MT, "one thread per bin");
  gbin[tid] = 0;
  __syncthreads();
  unsigned long long key[QF / MT];
  int bin[QF / MT];
#pragma unroll
  for (int u = 0; u < QF / MT; ++u) {
    const int i = tid + u * MT;
    bin[u] = -1;
    if (i < n) {
      const uint32_t b = (uint32_t)a.q[2 * (row0 + i) + 1] & hmask;
      key[u] = ((unsigned long long)b << 32) | (uint32_t)a.q[2 * (row0 + i)];
      bin[u] = (int)((b * 0x9E3779B1u) >> 22);
      atomicAdd(&gbin[bin[u]], 1);
    }
  }
  __syncthreads();
  {
    const int c = gbin[tid];
    const int incl = block_scan_incl(c, fs.wsum);       // (barriers inside)
    gbin[tid] = incl - c;                               // start of the bin
  }
  __syncthreads();
#pragma unroll
  for (int u = 0; u < QF / MT; ++u)
    if (bin[u] >= 0) qkeys[atomicAdd(&gbin[bin[u]], 1)] = key[u];
  __syncthreads();                                      // gbin[t] is now the END of bin t
  {
    const int lo = tid ? gbin[tid - 1] : 0, hi = gbin[tid];
    for (int i = lo + 1; i < hi; ++i) {                 // insertion sort of a few keys
      const unsigned long long x = qkeys[i];
      int j = i;
      while (j > lo && qkeys[j - 1] > x) { qkeys[j] = qkeys[j - 1]; --j; }
      qkeys[j] = x;
    }
  }
  __syncthreads();
  int base = 0;
  for (int i0 = 0; i0 < n; i0 += MT) {
    const int i = i0 + tid;
    uint32_t b = 0;
    int flag = 0;
    if (i < n) {
      b = (uint32_t)(qkeys[i] >> 32);
      flag = (i == 0 || (uint32_t)(qkeys[i - 1] >> 32) != b) ? 1 : 0;
    }
    const int incl = block_scan_incl(flag, fs.wsum);
    if (flag) {
      int m = 1;
      while (i + m < n && (uint32_t)(qkeys[i + m] >> 32) == b) ++m;
      const int g = base + incl - 1;
      hpos[g] = (unsigned short)i;
      hm[g] = (unsigned short)m;
      hn[g] = (unsigned short)min(a.depth, a.counts[b]);
      atomicMax(&fs.mmax, (unsigned)m);
    }
    base += fs.wsum[NW - 1];
  }
  __syncthreads();
  return base;
}

// One pass over the table entries the chunk's bucket groups select.
//   PASS 1: mark ids in the "seen" bitmap; ids seen before (or probed > threshcount times at once) join the set
//   PASS 2: entries whose id is a member (bitmap test, then set lookup) append their hits
//   PASS 3: admit single-record ids whose weight outranks (wk, idk)
template <int PASS>
__device__ void scan_chunk(const MatchArgs& a, FastShared& fs, unsigned char* smem, int G, uint2* mhits,
                           unsigned long long wk, unsigned idk, int nbase) {
  unsigned* bm = reinterpret_cast<unsigned*>(smem + OFF_R0);
  unsigned* mkeys = reinterpret_cast<unsigned*>(smem + OFF_MKEYS);
  unsigned* sid = reinterpret_cast<unsigned*>(smem + OFF_SID);
  unsigned* sraw = reinterpret_cast<unsigned*>(smem + OFF_SRAW);
  unsigned long long* sw = reinterpret_cast<unsigned long long*>(smem + OFF_SW);
  const unsigned long long* qkeys = reinterpret_cast<const unsigned long long*>(smem + OFF_Q);
  const unsigned short* hpos = reinterpret_cast<const unsigned short*>(smem + OFF_HPOS);
  const unsigned short* hm = hpos + QF;
  const unsigned short* hn = hm + QF;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t tmask = (1u << a.mtb) - 1u;
  const unsigned lt_mask = (1u << lane) - 1u;
  const double wk_d = __longlong_as_double((long long)wk);
  const int wcap = a.mh_cap / NW;                     // pass 2: hits this warp may append
  int wcount = PASS == 2 ? fs.wcount[warp] : 0;

  uint32_t nv[4] = {0u, 0u, 0u, 0u};
  auto fetch = [&](int g, uint32_t (&v)[4]) {          // first 128 slots of group g
    const int n = hn[g];
    const uint32_t* row = a.table + (size_t)(uint32_t)(qkeys[hpos[g]] >> 32) * a.depth;
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = (32 * u + lane < n) ? row[32 * u + lane] : 0u;
  };
  auto wanted = [&](int g) {                          // pass 3 reads only groups that could matter
    if (PASS != 3) return true;
    return a.hmin == 0u || (double)hm[g] / (double)a.hmin >= wk_d;
  };
  int g = warp;
  while (g < G && !wanted(g)) g += NW;
  if (g < G) fetch(g, nv);
  while (g < G) {
    uint32_t v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = nv[u];
    int gn = g + NW;
    while (gn < G && !wanted(gn)) gn += NW;
    if (gn < G) fetch(gn, nv);                          // in flight while this group is processed
    const int r = hpos[g], m = hm[g], n = hn[g];
    const uint32_t* row = a.table + (size_t)(uint32_t)(qkeys[r] >> 32) * a.depth;
    for (int s0 = 0; s0 < n; s0 += 128) {
      if (s0 > 0) {
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = (s0 + 32 * u + lane < n) ? row[s0 + 32 * u + lane] : 0u;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (s0 + 32 * u >= n) break;                    // warp-uniform
        const bool live = s0 + 32 * u + lane < n;
        const uint32_t id = (v[u] >> a.mtb) - 1u;
        const bool ok = live && id < (uint32_t)a.nids;
        if (PASS == 1) {
          if (ok) {
            const unsigned h = bm_index(id, a.bm_exact);
            const unsigned bit = 1u << (h & 31u);
            const unsigned old = atomicOr(&bm[h >> 5], bit);
            if ((old & bit) || m > a.thresh) {
              // join the member set; a probe sequence of PROBE_MAX means the set is (nearly) full:
              // the query is handed over (the members are counted after the pass)
              const unsigned key = id + 1u;
              unsigned s = set_hash(id);
              int tries = 0;
              while (true) {
                const unsigned k = atomicCAS(&mkeys[s], 0u, key);
                if (k == 0u || k == key) break;
                if (++tries >= PROBE_MAX) { fs.overflow = FS_SET_FULL; break; }
                s = (s + 1u) & (MSLOTS - 1);
              }
            }
          }
        } else if (PASS == 2) {
          int slot = -1;
          if (ok) {
            const unsigned h = bm_index(id, a.bm_exact);
            if ((bm[h >> 5] >> (h & 31u)) & 1u) slot = set_find(mkeys, id);
          }
          // every member entry appends its m hits; m is the same for the whole group, so the
          // positions come from one ballot and one atomic per warp
          const unsigned mem = __ballot_sync(0xffffffffu, slot >= 0);
          if (mem) {                                    // this warp's own segment of the list: no atomics
            const int total = __popc(mem) * m;
            if (wcount + total > wcap) {
              fs.overflow = FS_HITS_FULL;
            } else if (slot >= 0) {
              const int rt = (int)(v[u] & tmask) + a.bias;
              uint2* dst = mhits + (size_t)warp * wcap + wcount + __popc(mem & lt_mask) * m;
              for (int k = 0; k < m; ++k)
                dst[k] = make_uint2((unsigned)slot, (unsigned)(rt - (int)(uint32_t)qkeys[r + k]));
            }
            wcount += total;
          }
        } else {
          if (ok && set_find(mkeys, id) < 0) {
            const unsigned long long wb =
                (unsigned long long)__double_as_longlong((double)m / (double)a.hpi[id]);
            if (key_gt(wb, id, wk, idk)) {
              const unsigned x = atomicAdd(&fs.nx, 1u);
              if (x >= (unsigned)XCAP || nbase + (int)x >= SCAP) {
                fs.overflow = FS_EXTRAS_FULL;
              } else {
                sid[nbase + x] = id;
                sraw[nbase + x] = (unsigned)m;
                sw[nbase + x] = wb;
              }
            }
          }
        }
      }
    }
    g = gn;
  }
  if (PASS == 2 && lane == 0) fs.wcount[warp] = min(wcount, wcap);
}

// descending sort of the first n <= SCAP entries of (sw, sid) with sraw carried along: padded
// with zero keys to a power of two, then a bitonic sort
__device__ void rank_sort(unsigned char* smem, int n) {
  unsigned* sid = reinterpret_cast<unsigned*>(smem + OFF_SID);
  unsigned* sraw = reinterpret_cast<unsigned*>(smem + OFF_SRAW);
  unsigned long long* sw = reinterpret_cast<unsigned long long*>(smem + OFF_SW);
  int n2 = 2;
  while (n2 < n) n2 <<= 1;
  for (int i = n + threadIdx.x; i < n2; i += MT) { sid[i] = 0u; sraw[i] = 0u; sw[i] = 0ull; }
  __syncthreads();
  bitonic_sort(
      n2, [&](int i, int l, int k) { return key_gt(sw[i], sid[i], sw[l], sid[l]) != ((i & k) == 0); },
      [&](int i, int l) {
        const unsigned long long tw = sw[i]; sw[i] = sw[l]; sw[l] = tw;
        const unsigned ti = sid[i]; sid[i] = sid[l]; sid[l] = ti;
        const unsigned tr = sraw[i]; sraw[i] = sraw[l]; sraw[l] = tr;
      });
}

__global__ void __launch_bounds__(MT) afp_match_fast_kernel(MatchArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ FastShared fs;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  unsigned* bm = reinterpret_cast<unsigned*>(smem + OFF_R0);
  unsigned* mkeys = reinterpret_cast<unsigned*>(smem + OFF_MKEYS);
  unsigned* mcnt = reinterpret_cast<unsigned*>(smem + OFF_MCNT);
  int* whist = reinterpret_cast<int*>(smem + OFF_WH);
  unsigned* sid = reinterpret_cast<unsigned*>(smem + OFF_SID);
  unsigned* sraw = reinterpret_cast<unsigned*>(smem + OFF_SRAW);
  unsigned long long* sw = reinterpret_cast<unsigned long long*>(smem + OFF_SW);
  int* loff = reinterpret_cast<int*>(smem + OFF_LOFF);
  int* cur = reinterpret_cast<int*>(smem + OFF_CUR);
  unsigned char* pass = smem + OFF_PASS;
  unsigned short* map16 = reinterpret_cast<unsigned short*>(smem + OFF_MAP);
  uint2* mhits = a.mhits + (size_t)blockIdx.x * a.mh_cap;
  uint32_t* dts = a.dts + (size_t)blockIdx.x * a.hits_cap;
  int32_t* hist = a.hist + (size_t)blockIdx.x * a.hist_len;
  int32_t* filt = a.filt + (size_t)blockIdx.x * a.hist_len;
  auto zero_r0 = [&](int bytes) {
    uint4* z = reinterpret_cast<uint4*>(smem + OFF_R0);
    for (int i = tid; i < bytes / 16; i += MT) z[i] = make_uint4(0u, 0u, 0u, 0u);
  };

  for (int qi = blockIdx.x; qi < a.nqueries; qi += gridDim.x) {
    if (a.qskip && a.qskip[qi]) continue;          // (uniform) the long-query path takes it
    const int64_t q0 = a.qoff[qi];
    const int nq = (int)(a.qoff[qi + 1] - q0);
    __syncthreads();                               // the previous query is completely done
    if (tid == 0) {
      fs.nmem = 0; fs.nmh = 0; fs.nx = 0; fs.nabove = 0; fs.ndist = 0; fs.mmax = 0; fs.ngath = 0;
      fs.overflow = 0; fs.ms.nrows = 0;
    }
    if (tid < NW) fs.wcount[tid] = 0;
    zero_r0((BM_WORDS + MSLOTS) * 4);              // the "seen" bitmap and the member keys
    __syncthreads();
    int handover = FS_DONE;
    int K = 0, nabove = 0;
    const bool single = nq <= QF;                  // one sorted chunk stays in R2 for all passes
    int G1 = 0;
    if (nq > 0) {
      // ---- pass 1: which ids are hit by more than one (bucket, slot) record ----------------
      for (int c0 = 0; c0 < nq; c0 += QF) {
        G1 = prepare_chunk(a, fs, smem, q0 + c0, min(QF, nq - c0));
        scan_chunk<1>(a, fs, smem, G1, mhits, 0ull, 0u, 0);
        __syncthreads();
      }
      if (a.publish && a.bm_exact) {               // #distinct ids = bits set (exact bitmap only)
        int c = 0;
        for (int i = tid; i < BM_WORDS; i += MT) c += __popc(bm[i]);
        c = __reduce_add_sync(0xffffffffu, c);
        if (lane == 0 && c) atomicAdd(&fs.ndist, (unsigned)c);
      }
      __syncthreads();
      handover = fs.overflow;
      __syncthreads();
      if (!handover) {
        // ---- "member" bitmap, then pass 2: the hits of the members ---------------------------
        zero_r0(BM_WORDS * 4);
        __syncthreads();
        unsigned nm = 0;
        for (int s = tid; s < MSLOTS; s += MT) {
          const unsigned key = mkeys[s];
          if (key) {
            const unsigned h = bm_index(key - 1u, a.bm_exact);
            atomicOr(&bm[h >> 5], 1u << (h & 31u));
            ++nm;
          }
        }
        nm = __reduce_add_sync(0xffffffffu, nm);
        if (lane == 0 && nm) atomicAdd(&fs.nmem, nm);
        __syncthreads();
        if (fs.nmem > (unsigned)MMAX) handover = FS_SET_FULL;      // (uniform)
      }
      if (!handover) {
        for (int c0 = 0; c0 < nq; c0 += QF) {
          const int G = single ? G1 : prepare_chunk(a, fs, smem, q0 + c0, min(QF, nq - c0));
          scan_chunk<2>(a, fs, smem, G, mhits, 0ull, 0u, 0);
          __syncthreads();
        }
        handover = fs.overflow;
        if (tid == 0) {
          unsigned t = 0;
          for (int w = 0; w < NW; ++w) t += (unsigned)fs.wcount[w];
          fs.nmh = t;
        }
        __syncthreads();
      }
      int M = 0;                                   // entries in the rank arrays
      if (!handover) {
        // ---- exact raw counts = histogram of the member-hit list over the set slots ----------
        zero_r0((MSLOTS + WBINS) * 4);             // counters + weight histogram
        __syncthreads();
        {
          const int wcap = a.mh_cap / NW, n = fs.wcount[warp];
          const uint2* seg = mhits + (size_t)warp * wcap;
          for (int i = lane; i < n; i += 32) atomicAdd(&mcnt[seg[i].x], 1u);
        }
        __syncthreads();
        // ---- select: histogram of the weights' float image, #ids above threshcount -----------
        unsigned above = 0;
        for (int s = tid; s < MSLOTS; s += MT) {
          const unsigned key = mkeys[s];
          if (key) {
            const unsigned raw = mcnt[s];
            atomicAdd(&whist[weight_bin((double)raw / (double)a.hpi[key - 1u])], 1);
            above += raw > (unsigned)a.thresh ? 1u : 0u;
          }
        }
        above = __reduce_add_sync(0xffffffffu, above);
        if (lane == 0 && above) atomicAdd(&fs.nabove, above);
        __syncthreads();
        nabove = (int)fs.nabove;
        const int nmem = (int)fs.nmem;
        // candidate depth (audfprint_match.py:142-144); a table shard publishes its local
        // top-search_depth list instead
        if (a.publish) {
          if (a.bm_exact) K = min((int)fs.ndist, a.sdepth);
          else if (nmem >= a.sdepth) K = a.sdepth;
          else handover = FS_NDIST_UNKNOWN;        // #distinct ids unknown under a hashed bitmap
        } else {
          K = min(nabove, a.sdepth);
        }
        if (K > KCAP) handover = FS_DEPTH;
        if (!handover && K > 0) {
          // bin of the K-th largest weight: everything in a higher bin is in, that bin is undecided
          if (warp == 0) {
            constexpr int PER = WBINS / 32;
            int part = 0;
            for (int b = 0; b < PER; ++b) part += whist[lane * PER + b];
            int suffix = part;                       // members in lanes >= this one
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
              const int t = __shfl_down_sync(0xffffffffu, suffix, o);
              if (lane + o < 32) suffix += t;
            }
            const int need = min(K, nmem);
            const unsigned has = __ballot_sync(0xffffffffu, suffix >= need);
            const int L = 31 - __clz(has);           // highest lane whose suffix reaches `need`
            if (lane == L) {
              int cum = suffix - part;               // members in higher lanes
              int b = PER - 1;
              for (; b > 0; --b) {
                if (cum + whist[lane * PER + b] >= need) break;
                cum += whist[lane * PER + b];
              }
              fs.cut_bin = lane * PER + b;
              fs.cut_above = cum;
            }
          }
          __syncthreads();
          const int cut = fs.cut_bin;
          __syncthreads();                           // whist is dead: the rank arrays take its place
          for (int s = tid; s < MSLOTS; s += MT) {
            const unsigned key = mkeys[s];
            if (key) {
              const unsigned raw = mcnt[s];
              const double w = (double)raw / (double)a.hpi[key - 1u];
              if (weight_bin(w) >= cut) {
                const unsigned p = atomicAdd(&fs.ngath, 1u);
                if (p < (unsigned)SCAP) {
                  sw[p] = (unsigned long long)__double_as_longlong(w);
                  sid[p] = key - 1u;
                  sraw[p] = raw;
                }
              }
            }
          }
          __syncthreads();
          M = (int)fs.ngath;
          if (M > SCAP - XCAP) handover = FS_TIES;   // one weight bin holds thousands of members
        }
        if (!handover && K > 0) {
          rank_sort(smem, M);
          // ---- can a single-record id outrank the K-th member?  Its weight is m / hashesperid
          // with m <= min(m_max, threshcount).
          const unsigned long long wk = K <= M ? sw[K - 1] : 0ull;
          const unsigned idk = K <= M ? sid[K - 1] : 0u;
          const double bound = a.hmin ? (double)min((int)fs.mmax, a.thresh) / (double)a.hmin : INFINITY;
          const bool pruned = K <= M && bound < __longlong_as_double((long long)wk);
          __syncthreads();
          if (!pruned) {
            for (int c0 = 0; c0 < nq; c0 += QF) {
              const int G = single ? G1 : prepare_chunk(a, fs, smem, q0 + c0, min(QF, nq - c0));
              scan_chunk<3>(a, fs, smem, G, mhits, wk, idk, M);
              __syncthreads();
            }
            handover = fs.overflow;
            const int X = (int)fs.nx;
            __syncthreads();
            if (!handover && X > 0) {
              M += X;
              rank_sort(smem, M);
            }
            if (!handover && K > M) handover = FS_INCONSISTENT;   // cannot happen
          }
        }
      }
      if (!handover && K > 0) {
        // ---- the top-K: publish, dt-list offsets of the row-capable candidates ---------------
        const CandArrays cands{sid, sraw, loff, cur, pass};
        unsigned id = 0, raw = 0;
        unsigned long long wb = 0ull;
        if (tid < K) { id = sid[tid]; raw = sraw[tid]; wb = sw[tid]; }
        const bool rowable = candidates_begin(a, qi, K, id, raw, wb, cands, fs.wsum);
        for (int i = tid; i < MSLOTS; i += MT) map16[i] = 0xffffu;
        __syncthreads();
        if (rowable) map16[set_find(mkeys, id)] = (unsigned short)tid;     // raw > threshcount: a member
        __syncthreads();
        // ---- route the member hits of the row-capable candidates to their dt lists ----------
        {
          const int wcap = a.mh_cap / NW, n = fs.wcount[warp];
          const uint2* seg = mhits + (size_t)warp * wcap;
          for (int i0 = 0; i0 < n; i0 += 128) {
            uint2 h4[4];
#pragma unroll
            for (int u = 0; u < 4; ++u)
              h4[u] = (i0 + 32 * u + lane < n) ? seg[i0 + 32 * u + lane] : make_uint2(0xffffffffu, 0u);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              if (h4[u].x == 0xffffffffu) continue;
              const unsigned j = map16[h4[u].x];
              if (j != 0xffffu) dts[loff[j] + atomicAdd(&cur[j], 1)] = h4[u].y;
            }
          }
        }
        __syncthreads();
        candidates_finish(a, qi, K, cands, dts, fs.ms, hist, filt);
      }
    }
    __syncthreads();
    if (tid == 0) {
      int32_t* st = a.fstat + (size_t)qi * 8;
      st[0] = handover; st[1] = (int)fs.nmem; st[2] = (int)fs.nmh; st[3] = (int)fs.nx;
      st[4] = K; st[5] = nabove; st[6] = (int)fs.mmax; st[7] = (int)fs.ndist;
      if (handover) a.qlist[atomicAdd(a.nlist, 1)] = qi;       // the general kernel takes this query
      else query_done(a, qi, fs.ms.nrows, K, nabove);
    }
  }
}

}  // namespace

cudaError_t afp_launch_match_fast(const MatchArgs& a, int nctas, cudaStream_t stream) {
  cudaError_t e = cudaFuncSetAttribute(afp_match_fast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FAST_SMEM);
  if (e != cudaSuccess) return e;
  afp_match_fast_kernel<<<nctas, MT, FAST_SMEM, stream>>>(a);
  return cudaGetLastError();
}
