// HashTable.merge (reference hash_table.py:291-323) on the device-resident table.
//
// The reference, for self.merge(ht): every entry of ht moves up by idoffset = len(self.names) <<
// maxtimebits (uint32 arithmetic); then, for every bucket b with ht.counts[b] != 0 IN ASCENDING
// ORDER, the pool is our first min(counts, depth) entries followed by ht's first
// min(ht.counts, ht.depth) entries, shifted:
//   fits (pool <= depth)  the pool goes to slots 0..len-1 (slots beyond keep what they held) and
//                         counts[b] = len(pool);
//   overflows             table[b] = np.random.permutation(pool)[:depth] and counts[b] += ht.counts[b]
//                         (both raw).
// Only overflowing buckets draw from NumPy's global MT19937, one bucket after the other, and how
// many words a bucket draws depends on its pool SIZE alone (Fisher-Yates with masked rejection,
// afp_np_permutation_replay below).  So:
//   1. the incoming table goes up as raw rows (the buckets this table has) with its counts -
//      afp_table_merge; afp_table_merge_device reads rows and counts where they already lie in
//      device memory (a table exported by afp_table_export, e.g. received from another GPU) and
//      copies only the counts to the host for the checks;
//   2. one warp per bucket classifies it: a fitting pool is appended in place (only slots at or
//      beyond our prefix are written), an overflowing bucket is flagged with its pool size; a scan
//      compacts the flagged buckets in ascending order and their pool sizes go to the host;
//   3. the host replays the permutations on index arrays chunk by chunk.  Each chunk's surviving
//      pool indices (uint16 while every pool has at most 65536 entries, else uint32) go up, one warp
//      per bucket gathers the new row into scratch and a second kernel writes it back and adds the
//      raw counts - on the stream, while the host draws the next chunk.
// No result depends on the order of atomics: the compaction is a scan and every bucket is one
// warp's.  Tests: tests/test_gpu_table_merge.py (host merge, tests/merge_reference.py's statement,
// the reference's table-ops fixture); tests/test_table_merge_cpu.py (the replay against
// np.random.permutation).
#include <algorithm>
#include <chrono>
#include <vector>
#include "afp_internal.cuh"

namespace {

constexpr int WARPS = 8;                           // buckets per 256-thread CTA
constexpr int64_t CHUNK_INDICES = (int64_t)1 << 22; // surviving indices replayed per pipeline step

struct MergeArgs {
  uint32_t* table;              // our table [nb][depth]
  int32_t* counts;              // [nb]
  int depth;
  const uint32_t* in_table;     // incoming rows [in_nb][in_depth] (only the buckets we have)
  const int32_t* in_counts;     // [in_nb]
  int in_depth;
  int64_t in_nb;
  uint32_t shift;               // idoffset
};

__device__ __forceinline__ int prefix_len(int32_t count, int depth) { return max(0, min(count, depth)); }

// per incoming bucket: append a fitting pool, or flag an overflowing one with its pool size
__global__ void __launch_bounds__(256) afp_merge_classify_kernel(MergeArgs a, int32_t* flag, int32_t* pool_of) {
  const int64_t b = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5);
  if (b >= a.in_nb) return;
  const int lane = threadIdx.x & 31;
  const int32_t cin = a.in_counts[b];
  int32_t pool = 0;
  if (cin != 0) {
    const int have = prefix_len(a.counts[b], a.depth);
    const int add = prefix_len(cin, a.in_depth);
    const int64_t p = (int64_t)have + add;
    if (p <= a.depth) {
      uint32_t* row = a.table + (size_t)b * a.depth;
      const uint32_t* in = a.in_table + (size_t)b * a.in_depth;
      for (int j = lane; j < add; j += 32) row[have + j] = in[j] + a.shift;
      if (lane == 0) a.counts[b] = (int32_t)p;
    } else {
      pool = (int32_t)p;
    }
  }
  if (lane == 0) {
    flag[b] = pool > 0 ? 1 : 0;
    pool_of[b] = pool;
  }
}

// overflowing buckets in ascending order, with their pool sizes
__global__ void afp_merge_compact_kernel(const int32_t* flag, const int32_t* pool_of, const int64_t* off, int64_t n,
                                         uint32_t* bkt, int32_t* psz) {
  const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n || !flag[b]) return;
  bkt[off[b]] = (uint32_t)b;
  psz[off[b]] = pool_of[b];
}

// one warp per overflowing bucket of a chunk: slot s of the new row = pool[idx[s]]
template <class IdxT>
__global__ void __launch_bounds__(256) afp_merge_gather_kernel(MergeArgs a, const uint32_t* bkt, int64_t n,
                                                               const IdxT* idx, uint32_t* out) {
  const int64_t o = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5);
  if (o >= n) return;
  const int lane = threadIdx.x & 31;
  const uint32_t b = bkt[o];
  const uint32_t* row = a.table + (size_t)b * a.depth;
  const uint32_t* in = a.in_table + (size_t)b * a.in_depth;
  const uint32_t have = (uint32_t)prefix_len(a.counts[b], a.depth);
  const IdxT* k = idx + (size_t)o * a.depth;
  uint32_t* dst = out + (size_t)o * a.depth;
  for (int s = lane; s < a.depth; s += 32) {
    const uint32_t j = k[s];
    dst[s] = j < have ? row[j] : in[j - have] + a.shift;
  }
}

__global__ void __launch_bounds__(256) afp_merge_writeback_kernel(MergeArgs a, const uint32_t* bkt, int64_t n,
                                                                  const uint32_t* src) {
  const int64_t o = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5);
  if (o >= n) return;
  const int lane = threadIdx.x & 31;
  const uint32_t b = bkt[o];
  uint32_t* row = a.table + (size_t)b * a.depth;
  const uint32_t* s = src + (size_t)o * a.depth;
  for (int j = lane; j < a.depth; j += 32) row[j] = s[j];
  if (lane == 0) a.counts[b] = (int32_t)((uint32_t)a.counts[b] + (uint32_t)a.in_counts[b]);   // wraps as int32 does
}

// ---- NumPy's legacy MT19937 (RandomState) --------------------------------------------------------
// state = np.random.get_state()[1:3]: 624 key words + the position.  next32 is numpy's
// mt19937_next32 (the same words as CPython's genrand_uint32 from the same state).
struct Mt {
  uint32_t mt[624];
  uint32_t pos;
  void refill() {
    constexpr int N = 624, M = 397;
    constexpr uint32_t A = 0x9908b0dfu, UP = 0x80000000u, LO = 0x7fffffffu;
    int k = 0;
    for (; k < N - M; ++k) {
      const uint32_t y = (mt[k] & UP) | (mt[k + 1] & LO);
      mt[k] = mt[k + M] ^ (y >> 1) ^ ((0u - (y & 1u)) & A);
    }
    for (; k < N - 1; ++k) {
      const uint32_t y = (mt[k] & UP) | (mt[k + 1] & LO);
      mt[k] = mt[k + (M - N)] ^ (y >> 1) ^ ((0u - (y & 1u)) & A);
    }
    const uint32_t y = (mt[N - 1] & UP) | (mt[0] & LO);
    mt[N - 1] = mt[M - 1] ^ (y >> 1) ^ ((0u - (y & 1u)) & A);
    pos = 0;
  }
  inline uint32_t next32() {
    if (pos >= 624u) refill();
    uint32_t y = mt[pos++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
  }
};

// RandomState.permutation(pool) of one 1-D pool of m entries, on the indices 0..m-1: the shuffle
// runs i = m-1 .. 1 and draws j = random_interval(i) (mask = next power of two of i, minus 1;
// redraw while (word & mask) > i), then swaps x[i], x[j].  The first `keep` indices are written.
template <class OutT>
inline void permute_one(Mt& g, uint32_t m, uint32_t keep, std::vector<uint32_t>& x, OutT* out) {
  if (x.size() < m) x.resize(m);
  uint32_t* v = x.data();
  for (uint32_t i = 0; i < m; ++i) v[i] = i;
  for (uint32_t i = m - 1; i >= 1; --i) {
    const uint32_t mask = 0xffffffffu >> __builtin_clz(i);
    uint32_t j;
    do j = g.next32() & mask; while (j > i);
    const uint32_t t = v[i];
    v[i] = v[j];
    v[j] = t;
  }
  for (uint32_t s = 0; s < keep; ++s) out[s] = (OutT)v[s];
}

double ms_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

// the overflowing buckets: replay chunk k on the host while the device applies chunk k - 1
template <class IdxT>
int apply_overflow(afp_ctx* c, const MergeArgs& a, const std::vector<int32_t>& psz, Mt& g, double* stage_ms) {
  const int64_t n = (int64_t)psz.size();
  const int64_t per = std::max<int64_t>(1, CHUNK_INDICES / a.depth);
  const size_t chunk_idx = (size_t)std::min(per, n) * (size_t)a.depth;
  AFP_CUDA(c, c->d_mg_idx.reserve(sizeof(IdxT) * chunk_idx));
  AFP_CUDA(c, c->d_mg_row.reserve(sizeof(uint32_t) * chunk_idx));
  std::vector<IdxT> h_idx(chunk_idx);
  std::vector<uint32_t> x;
  const uint32_t* bkt = c->d_mg_bkt.as<uint32_t>();
  std::vector<cudaEvent_t> ev;
  auto fail = [&](int rc) {
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
    return rc;
  };
  double replay_ms = 0.0;
  for (int64_t o0 = 0; o0 < n; o0 += per) {
    const int64_t m = std::min(per, n - o0);
    const auto t0 = std::chrono::steady_clock::now();
    for (int64_t o = 0; o < m; ++o)
      permute_one(g, (uint32_t)psz[(size_t)(o0 + o)], (uint32_t)a.depth, x, h_idx.data() + (size_t)o * a.depth);
    replay_ms += ms_since(t0);
    // pageable source: the copy returns once h_idx is staged, so it may be refilled right away
    cudaEvent_t e[3] = {};
    if (stage_ms) {
      for (auto& ei : e) {
        cudaError_t r = cudaEventCreate(&ei);
        if (r != cudaSuccess) {
          c->err = std::string("cudaEventCreate: ") + cudaGetErrorString(r);
          return fail(AFP_ERR_CUDA);
        }
        ev.push_back(ei);
      }
      cudaEventRecord(e[0], c->stream);
    }
    cudaError_t r = cudaMemcpyAsync(c->d_mg_idx.p, h_idx.data(), sizeof(IdxT) * (size_t)m * a.depth,
                                    cudaMemcpyHostToDevice, c->stream);
    if (r != cudaSuccess) {
      c->err = std::string("cudaMemcpyAsync (pool indices): ") + cudaGetErrorString(r);
      return fail(AFP_ERR_CUDA);
    }
    if (stage_ms) cudaEventRecord(e[1], c->stream);
    const unsigned grid = (unsigned)((m + WARPS - 1) / WARPS);
    int rc;
    if ((rc = afp_launch(c, afp_merge_gather_kernel<IdxT>, grid, 256, 0, a, bkt + o0, m, c->d_mg_idx.as<IdxT>(),
                         c->d_mg_row.as<uint32_t>())) ||
        (rc = afp_launch(c, afp_merge_writeback_kernel, grid, 256, 0, a, bkt + o0, m, c->d_mg_row.as<uint32_t>())))
      return fail(rc);
    if (stage_ms) cudaEventRecord(e[2], c->stream);
  }
  const auto t1 = std::chrono::steady_clock::now();
  cudaError_t r = cudaStreamSynchronize(c->stream);
  if (r != cudaSuccess) {
    c->err = std::string("cudaStreamSynchronize (merge apply): ") + cudaGetErrorString(r);
    return fail(AFP_ERR_CUDA);
  }
  if (stage_ms) {
    float up = 0.f, kern = 0.f;
    for (size_t i = 0; i < ev.size(); i += 3) {
      float t = 0.f;
      cudaEventElapsedTime(&t, ev[i], ev[i + 1]);
      up += t;
      cudaEventElapsedTime(&t, ev[i + 1], ev[i + 2]);
      kern += t;
    }
    stage_ms[2] = replay_ms;
    stage_ms[3] = up;
    stage_ms[4] = kern;
    stage_ms[5] = ms_since(t1);
  }
  return fail(AFP_OK);
}

// the checks both merge entries make before anything changes; `counts` is a HOST copy of the
// incoming counts [2^hashbits]
int merge_check(afp_ctx* c, const int32_t* counts, int32_t hashbits, int32_t depth, int64_t id_offset,
                const uint32_t* np_state625) {
  if (!c->tab.loaded) AFP_FAIL(c, AFP_ERR_STATE, "no table on the device");
  if (hashbits < 1 || hashbits > 28 || depth < 1) AFP_FAIL(c, AFP_ERR_INVALID, "bad geometry of the incoming table");
  if (np_state625[624] > 624u) AFP_FAIL(c, AFP_ERR_INVALID, "MT19937 position above 624");
  const int mtb = c->tab.maxtimebits;
  if (id_offset < 0 || (id_offset << mtb) >= ((int64_t)1 << 32))
    AFP_FAIL(c, AFP_ERR_INVALID, "id offset does not fit in 32 - maxtimebits bits");
  const int64_t nb = (int64_t)1 << c->tab.hashbits, in_nb = (int64_t)1 << hashbits;
  for (int64_t b = 0; b < in_nb; ++b) {
    if (counts[b] < 0) AFP_FAIL(c, AFP_ERR_INVALID, "negative count in the incoming table");
    if (b >= nb && counts[b] != 0)
      AFP_FAIL(c, AFP_ERR_INDEX, "a live bucket of the incoming table lies outside this table (hash_table.py:302)");
  }
  return AFP_OK;
}

// classify, compaction, replay and apply on incoming rows that are already on the device: d_in
// [nm][depth] rows of the incoming table (only the buckets we have), d_cnt [nm] its counts
int merge_body(afp_ctx* c, const uint32_t* d_in, const int32_t* d_cnt, int32_t depth, int64_t nm, int64_t id_offset,
               uint32_t* np_state625, int64_t* noverflow, double* stage_ms) {
  auto t0 = std::chrono::steady_clock::now();
  MergeArgs a;
  a.table = c->tab.table.as<uint32_t>(); a.counts = c->tab.counts.as<int32_t>(); a.depth = c->tab.depth;
  a.in_table = d_in; a.in_counts = d_cnt; a.in_depth = depth; a.in_nb = nm;
  a.shift = (uint32_t)(id_offset << c->tab.maxtimebits);
  AFP_CUDA(c, c->d_mg_off.reserve(sizeof(int64_t) * (size_t)(nm + 1)));
  int32_t *flag = nullptr, *pool_of = nullptr;
  int64_t* off = c->d_mg_off.as<int64_t>();
  int64_t n = 0;
  int rc;
  if ((rc = afp_carve(c, c->d_mg_flag, [&](Carver& k) {
         flag = k.take<int32_t>(nm);
         pool_of = k.take<int32_t>(nm);
       })) ||
      (rc = afp_launch(c, afp_merge_classify_kernel, (unsigned)((nm + WARPS - 1) / WARPS), 256, 0, a, flag, pool_of)) ||
      (rc = afp_scan_large(c, flag, off, nm)) || (rc = afp_read_back(c, &n, off + nm, 1)))
    return rc;
  std::vector<int32_t> psz((size_t)n);
  if (n > 0) {
    uint32_t* d_bkt = nullptr;
    int32_t* d_psz = nullptr;
    if ((rc = afp_carve(c, c->d_mg_bkt, [&](Carver& k) {
           d_bkt = k.take<uint32_t>(n);
           d_psz = k.take<int32_t>(n);
         })) ||
        (rc = afp_launch(c, afp_merge_compact_kernel, (unsigned)((nm + 255) / 256), 256, 0, flag, pool_of, off, nm,
                         d_bkt, d_psz)) ||
        (rc = afp_read_back(c, psz.data(), d_psz, (size_t)n)))
      return rc;
  }
  if (stage_ms) stage_ms[1] = ms_since(t0);
  if (n > 0) {
    Mt g;
    std::copy(np_state625, np_state625 + 624, g.mt);
    g.pos = np_state625[624];
    const int32_t pmax = *std::max_element(psz.begin(), psz.end());
    rc = pmax <= 65536 ? apply_overflow<uint16_t>(c, a, psz, g, stage_ms) : apply_overflow<uint32_t>(c, a, psz, g, stage_ms);
    if (rc) return rc;
    std::copy(g.mt, g.mt + 624, np_state625);
    np_state625[624] = g.pos;
  }
  if (noverflow) *noverflow = n;
  // the table now names ids the device's hashesperid does not have yet: no pruning until the
  // caller's afp_table_set_hashesperid recomputes the bound over the merged table
  c->tab.hmin = 0;
  return AFP_OK;
}

}  // namespace

extern "C" {

int afp_np_permutation_replay(uint32_t* state625, const int32_t* pool_sizes, int64_t n, int32_t keep,
                              int32_t* out) {
  if (!state625 || n < 0 || keep < 1 || (n > 0 && (!pool_sizes || !out))) return AFP_ERR_INVALID;
  if (state625[624] > 624u) return AFP_ERR_INVALID;
  for (int64_t i = 0; i < n; ++i)
    if (pool_sizes[i] < keep) return AFP_ERR_INVALID;          // nothing drawn yet: the state is unchanged
  Mt g;
  std::copy(state625, state625 + 624, g.mt);
  g.pos = state625[624];
  std::vector<uint32_t> x;
  for (int64_t i = 0; i < n; ++i) permute_one(g, (uint32_t)pool_sizes[i], (uint32_t)keep, x, out + (size_t)i * keep);
  std::copy(g.mt, g.mt + 624, state625);
  state625[624] = g.pos;
  return AFP_OK;
}

int afp_table_merge(afp_ctx* c, const uint32_t* table, const int32_t* counts, int32_t hashbits, int32_t depth,
                    int64_t id_offset, uint32_t* np_state625, int64_t* noverflow, double* stage_ms) {
  if (!c || !table || !counts || !np_state625) return AFP_ERR_INVALID;
  int rc = merge_check(c, counts, hashbits, depth, id_offset, np_state625);
  if (rc) return rc;
  const int64_t nm = std::min((int64_t)1 << c->tab.hashbits, (int64_t)1 << hashbits);
  if (noverflow) *noverflow = 0;
  if (stage_ms) std::fill(stage_ms, stage_ms + 6, 0.0);
  AFP_CUDA(c, cudaSetDevice(c->device));
  const auto t0 = std::chrono::steady_clock::now();
  uint32_t* d_in = nullptr;
  int32_t* d_cnt = nullptr;
  if ((rc = afp_carve(c, c->d_mg_in, [&](Carver& k) {
         d_in = k.take<uint32_t>(nm * depth);
         d_cnt = k.take<int32_t>(nm);
       })))
    return rc;
  AFP_CUDA(c, afp_copy_in(c, d_in, table, (size_t)nm * depth, 1));
  AFP_CUDA(c, afp_copy_in(c, d_cnt, counts, (size_t)nm, 1));
  if (stage_ms) {
    AFP_CUDA(c, cudaStreamSynchronize(c->stream));
    stage_ms[0] = ms_since(t0);
  }
  return merge_body(c, d_in, d_cnt, depth, nm, id_offset, np_state625, noverflow, stage_ms);
}

int afp_table_merge_device(afp_ctx* c, const uint32_t* table_dev, const int32_t* counts_dev, int32_t hashbits,
                           int32_t depth, int64_t id_offset, uint32_t* np_state625, int64_t* noverflow,
                           double* stage_ms) {
  if (!c || !table_dev || !counts_dev || !np_state625) return AFP_ERR_INVALID;
  if (hashbits < 1 || hashbits > 28 || depth < 1) AFP_FAIL(c, AFP_ERR_INVALID, "bad geometry of the incoming table");
  AFP_CUDA(c, cudaSetDevice(c->device));
  // the checks read the counts on the host (4 MB at 2^20 buckets); the rows stay where they are
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<int32_t> h_counts((size_t)1 << hashbits);
  int rc = afp_read_back(c, h_counts.data(), counts_dev, h_counts.size());
  if (rc) return rc;
  const double download_ms = ms_since(t0);
  rc = merge_check(c, h_counts.data(), hashbits, depth, id_offset, np_state625);
  if (rc) return rc;
  if (noverflow) *noverflow = 0;
  if (stage_ms) {
    std::fill(stage_ms, stage_ms + 6, 0.0);
    stage_ms[0] = download_ms;
  }
  const int64_t nm = std::min((int64_t)1 << c->tab.hashbits, (int64_t)1 << hashbits);
  return merge_body(c, table_dev, counts_dev, depth, nm, id_offset, np_state625, noverflow, stage_ms);
}

int afp_table_export(afp_ctx* c, uint32_t* table_dev, int32_t* counts_dev) {
  if (!c || !table_dev || !counts_dev) return AFP_ERR_INVALID;
  if (!c->tab.loaded) AFP_FAIL(c, AFP_ERR_STATE, "no table on the device");
  AFP_CUDA(c, cudaSetDevice(c->device));
  const size_t nb = (size_t)1 << c->tab.hashbits;
  AFP_CUDA(c, afp_copy_out(c, table_dev, c->tab.table.as<uint32_t>(), nb * (size_t)c->tab.depth, 0));
  AFP_CUDA(c, afp_copy_out(c, counts_dev, c->tab.counts.as<int32_t>(), nb, 0));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  return AFP_OK;
}

}  // extern "C"
