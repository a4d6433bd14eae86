// K2 — onset high-pass + forward/backward decaying-threshold peak picking (FP64).
//
// Replaces, per item (file x shift), the rest of Analyzer.find_peaks:
//   per-bin lfilter([1,-1],[1,-0.98])                 audfprint_analyze.py:293-295
//   locmax                                             :36-52
//   spreadpeaksinvector / spreadpeaks                  :153-197
//   _decaying_threshold_fwd_prune                      :199-231
//   _decaying_threshold_bwd_prune_peaks                :233-253
//   peak list build (column-major, bins ascending)     :303-308
//
// The time recursion is strictly sequential inside an item, so the unit of
// parallelism is ONE WARP PER ITEM (one warp per CTA): lane l owns bins
// 8l..8l+7 (threshold, filter state and the current column live in registers), the column stream arrives through a TMA bulk-copy ring in shared
// memory (2 chunks of 4 columns per warp), neighbour compares use warp
// shuffles, the per-column top-N selection uses redux.sync (warp-wide integer
// max on the bit pattern of the positive doubles), and thousands of items run
// concurrently.  All arithmetic that feeds a comparison is done with explicit
// round-to-nearest FP64 intrinsics (no FMA contraction) in the operation order
// of the reference, so given the same spectrogram the decisions are bit-exact.
#include <math.h>
#include "afp_internal.cuh"
#include "afp_tma.cuh"

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int CH = 4;      // columns per TMA chunk (8 KB)
constexpr int NST = 2;     // chunks in flight per warp (16 KB ring)
constexpr int PFB = 8;     // prefetch distance (columns) of the backward pass

// K2 is one warp per item and every item lasts about T column steps, so the kernel takes as many
// item-durations as it has waves: the whole default batch (1024 items) has to be resident at once.
// 10 CTAs per SM (1320 on a 132-SM H100 SXM, 1140 on a 114-SM H100 PCIe) leave 233,472 / 10 B of
// shared memory per CTA, of which the runtime reserves 1 KB.
constexpr int K2_CTAS_PER_SM = 10;
constexpr size_t K2_SMEM_BUDGET = 233472 / K2_CTAS_PER_SM - 1024;
constexpr size_t k2_static_smem(size_t rsize) {
  return sizeof(double) * AFP_GAUSS_PAD + 128 /* sCol alignment */ + NST * CH * AFP_NBINS * rsize +
         NST * sizeof(unsigned long long);
}
static_assert(k2_static_smem(sizeof(double)) <= K2_SMEM_BUDGET,
              "K2's shared memory would fit fewer than 10 CTAs per SM: a 1024-item batch would run in two waves");

struct PeakArgs {
  const ItemDesc* items;
  const ItemStats* stats;
  int item0;
  const void* logs;       // [frames][256], double (default) or float (FP32 spectrogram mode)
  const double* gauss;    // AFP_GAUSS_N
  double a_dec, pole;
  int maxpks;
  double* fwd_val;        // [frames][maxpks]
  uint8_t* fwd_bin;       // [frames][maxpks]
  uint8_t* fwd_cnt;       // [frames]
  uint8_t* pk_bin;        // [frames][maxpks]
  uint8_t* pk_cnt;        // [frames]
  int32_t* item_scols;
  int32_t* item_npeaks;
};

// Lane l owns the 8 contiguous bins 8l..8l+7 (register j = bin & 7): the local-max test
// then needs only one neighbour exchange per side.  The Gaussian table is stored with one
// pad element per 8 (index k + k/8) so that the lanes' 64-byte-strided reads hit distinct banks.
__device__ __forceinline__ int bin_of(int lane, int j) { return 8 * lane + j; }
__device__ __forceinline__ int lane_of(int pos) { return pos >> 3; }
__device__ __forceinline__ int reg_of(int pos) { return pos & 7; }
__device__ __forceinline__ int gidx(int k) { return k + (k >> 3); }   // padded table index

// thr = max(thr, val * E[bin - pos]) for the 8 bins of this lane
// (audfprint_analyze.py:225-227 / :193-196).
// A threshold starts at 0 and is only ever raised by max() or scaled by a_dec > 0, so it is
// never NaN: compare-and-select then makes the same decisions as fmax(), without its NaN fix-up.
// The 8 entries are consecutive in the table; in its padded layout those from the next group
// of 8 on sit one element further, so two base addresses serve all 8 loads.
__device__ __forceinline__ void bump(double (&thr)[8], const double* sE, int lane, int pos, double val) {
  const int k0 = AFP_NBINS - pos + 8 * lane;
  const uint32_t e0 = smem_u32(sE + gidx(k0)), e1 = e0 + 8;
  const int split = 8 - (k0 & 7);   // gidx(k0 + j) == gidx(k0) + j + (j >= split)
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    double e;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(e) : "r"((j >= split ? e1 : e0) + 8 * j) : "memory");
    const double p = __dmul_rn(val, e);
    thr[j] = p > thr[j] ? p : thr[j];
  }
}

__device__ __forceinline__ double pick(const double (&v)[8], int j) {
  double x = v[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) x = (j == i) ? v[i] : x;
  return x;
}

// locmax (audfprint_analyze.py:36-52): bit j set iff bin 8*lane+j is a local max
__device__ __forceinline__ unsigned locmax_mask(const double (&s)[8], int lane) {
  const double left = __shfl_up_sync(FULL, s[7], 1);
  const double right = __shfl_down_sync(FULL, s[0], 1);
  bool ge[9];
  ge[0] = (lane == 0) ? true : (s[0] >= left);
#pragma unroll
  for (int j = 1; j < 8; ++j) ge[j] = s[j] >= s[j - 1];
  ge[8] = (lane == 31) ? false : (right >= s[7]);
  unsigned m = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) m |= (ge[j] && !ge[j + 1]) ? (1u << j) : 0u;
  return m;
}

// spreadpeaksinvector (audfprint_analyze.py:153-160): start from zeros, lay a
// Gaussian on every local max of v.
__device__ __forceinline__ void spread(const double (&v)[8], double (&thr)[8], const double* sE, int lane) {
#pragma unroll
  for (int j = 0; j < 8; ++j) thr[j] = 0.0;
  const unsigned m = locmax_mask(v, lane);
  unsigned lanes = __ballot_sync(FULL, m != 0);
  while (lanes) {
    const int src = __ffs(lanes) - 1;
    lanes &= lanes - 1;
    unsigned mm = __shfl_sync(FULL, m, src);
    while (mm) {
      const int j = __ffs(mm) - 1;
      mm &= mm - 1;
      const double val = __shfl_sync(FULL, pick(v, j), src);
      bump(thr, sE, lane, bin_of(src, j), val);
    }
  }
}

// floor, mean removal and one step of the DF2T high-pass
// y = z + x ; z = -x + pole*y   (scipy lfilter order, SURVEY.md §8c)
__device__ __forceinline__ void hpf_step(const double (&l)[8], double (&z)[8], double (&s)[8], double lf,
                                         double mean, double pole) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const double x = __dsub_rn(fmax(l[j], lf), mean);
    const double y = __dadd_rn(z[j], x);
    z[j] = __dadd_rn(-x, __dmul_rn(pole, y));
    s[j] = y;
  }
}

// The column stream of one item: chunks of CH columns are TMA-bulk-copied into a ring of
// NST shared-memory stages (one mbarrier each), NST chunks ahead of the consumer.
template <typename R>
struct ColRing {
  R* buf;                      // NST * CH * 256 values
  unsigned long long* bar;     // NST mbarriers
  const R* src;                // column 0 of the item
  int T;
  int lane;

  __device__ __forceinline__ void issue(int chunk) const {   // lane 0 only
    const int c0 = chunk * CH;
    const uint32_t bytes = (uint32_t)min(CH, T - c0) * AFP_NBINS * sizeof(R);
    bulk_copy_g2s(buf + (chunk % NST) * CH * AFP_NBINS, src + (size_t)c0 * AFP_NBINS, bytes, bar + (chunk % NST));
  }
  __device__ __forceinline__ void wait(int chunk) const { mbar_wait(bar + (chunk % NST), (chunk / NST) & 1); }
  // this lane's 8 values of one column (shared or global memory)
  __device__ __forceinline__ void read(const R* col, double (&x)[8]) const {
    if (sizeof(R) == 8) {
      const double2* p = reinterpret_cast<const double2*>(col) + 4 * lane;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const double2 v = p[i];
        x[2 * i] = v.x;
        x[2 * i + 1] = v.y;
      }
    } else {
      const float4* p = reinterpret_cast<const float4*>(col) + 2 * lane;
      const float4 u = p[0], v = p[1];
      x[0] = u.x; x[1] = u.y; x[2] = u.z; x[3] = u.w;
      x[4] = v.x; x[5] = v.y; x[6] = v.z; x[7] = v.w;
    }
  }
  // column t straight from global memory, bypassing the ring
  __device__ __forceinline__ void peek(int t, double (&x)[8]) const { read(src + (size_t)t * AFP_NBINS, x); }
  // column t from the ring; the chunk is recycled after its last column
  __device__ __forceinline__ void load(int t, double (&x)[8]) const {
    const int chunk = t / CH;
    if (t % CH == 0) wait(chunk);
    read(buf + ((chunk % NST) * CH + t % CH) * AFP_NBINS, x);
    if (t % CH == CH - 1 || t == T - 1) {
      __syncwarp();
      if (lane == 0 && (chunk + NST) * CH < T) issue(chunk + NST);
    }
  }
};

template <typename R>
__global__ void __launch_bounds__(32) afp_peaks_kernel(PeakArgs a) {
  __shared__ __align__(16) double sE[AFP_GAUSS_PAD];
  __shared__ __align__(128) R sCol[NST * CH * AFP_NBINS];
  __shared__ unsigned long long sBar[NST];
  const int lane = threadIdx.x;
  const int item = a.item0 + blockIdx.x;
  for (int k = lane; k < AFP_GAUSS_N; k += 32) sE[gidx(k)] = a.gauss[k];

  const ItemDesc it = a.items[item];
  const ItemStats st = a.stats[item];
  const int T = it.nframes;
  const int64_t base = it.frame_base;
  const int maxpks = a.maxpks;
  if (T == 0 || st.allzero) {
    // identically-zero input: sgram stays 0, nothing exceeds the (zero) threshold
    for (int t = lane; t < T; t += 32) a.pk_cnt[base + t] = 0;
    if (lane == 0) {
      a.item_scols[item] = 0;
      a.item_npeaks[item] = 0;
    }
    return;
  }
  ColRing<R> ring{sCol, sBar, reinterpret_cast<const R*>(a.logs) + base * AFP_NBINS, T, lane};
  if (lane == 0) {
    mbar_init<NST>(sBar);
    for (int c = 0; c < NST && c * CH < T; ++c) ring.issue(c);
  }
  __syncwarp();
  const double lf = st.logfloor, mean = st.mean, pole = a.pole, a_dec = a.a_dec;

  double thr[8], z[8], s[8], sn[8], l[8];

  // ---- initial threshold: spread of the per-bin max over the first 10 columns
  // (audfprint_analyze.py:204-206), read from global memory while the ring fills with columns
  // 0..NST*CH-1 for the forward pass (the ring is smaller than 10 columns)
  {
    double mx[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { z[j] = 0.0; mx[j] = -INFINITY; }
    const int n0 = min(10, T);
    for (int t = 0; t < n0; ++t) {
      ring.peek(t, l);
      hpf_step(l, z, s, lf, mean, pole);
#pragma unroll
      for (int j = 0; j < 8; ++j) mx[j] = fmax(mx[j], s[j]);
    }
    spread(mx, thr, sE, lane);
  }

  // ---- forward pass (audfprint_analyze.py:214-230) ------------------------------
  // Software pipeline: column t+1 is high-passed and local-max'ed (independent of
  // the threshold) before the threshold-dependent decisions of column t.
#pragma unroll
  for (int j = 0; j < 8; ++j) z[j] = 0.0;
  ring.load(0, l);
  hpf_step(l, z, s, lf, mean, pole);
  unsigned lm = locmax_mask(s, lane);
  for (int t = 0; t < T; ++t) {
    unsigned lmn = 0;
    if (t + 1 < T) {
      ring.load(t + 1, l);
      hpf_step(l, z, sn, lf, mean, pole);
      lmn = locmax_mask(sn, lane);
    }
    unsigned cmask = lm;
#pragma unroll
    for (int j = 0; j < 8; ++j) cmask &= (s[j] > thr[j]) ? ~0u : ~(1u << j);
    int npk = 0;
    if (__ballot_sync(FULL, cmask != 0)) {
      // accept candidates by (value desc, bin desc) (:220), at most maxpks (:221)
      while (true) {
        unsigned long long bk = 0ull;
        int bj = -1;
#pragma unroll
        for (int j = 0; j < 8; ++j) {   // bins ascend with j inside a lane: >= keeps the higher bin on ties
          const unsigned long long k = (unsigned long long)__double_as_longlong(s[j]);
          if (((cmask >> j) & 1u) && k >= bk) { bk = k; bj = j; }
        }
        const unsigned hi = (unsigned)(bk >> 32), lo = (unsigned)bk;
        const unsigned mhi = __reduce_max_sync(FULL, bj >= 0 ? hi : 0u);
        const bool v1 = bj >= 0 && hi == mhi;
        const unsigned mlo = __reduce_max_sync(FULL, v1 ? lo : 0u);
        const bool v2 = v1 && lo == mlo;
        const int pos = (int)__reduce_max_sync(FULL, v2 ? (unsigned)(bin_of(lane, bj) + 1) : 0u) - 1;
        const double val = __longlong_as_double((long long)(((unsigned long long)mhi << 32) | mlo));
        if (lane == lane_of(pos)) cmask &= ~(1u << reg_of(pos));
        bump(thr, sE, lane, pos, val);
        if (lane == 0) {
          a.fwd_val[(base + t) * maxpks + npk] = val;
          a.fwd_bin[(base + t) * maxpks + npk] = (uint8_t)pos;
        }
        ++npk;
        if (npk >= maxpks || !__ballot_sync(FULL, cmask != 0)) break;
      }
    }
    if (lane == 0) a.fwd_cnt[base + t] = (uint8_t)npk;
#pragma unroll
    for (int j = 0; j < 8; ++j) thr[j] = __dmul_rn(thr[j], a_dec);
    if (t + 1 < T) {
#pragma unroll
      for (int j = 0; j < 8; ++j) s[j] = sn[j];
      lm = lmn;
    }
  }
  __syncwarp();   // make lane 0's fwd_* stores visible to the whole warp

  // ---- backward pass (audfprint_analyze.py:233-253) ----------------------------
  spread(s, thr, sE, lane);   // s still holds the last column (:237)
  int nxt_bin = -1, nxt_alive = 0;
  int scols = 0, npeaks = 0;
  // emit the final peaks of one column: bins ascending (:303-308)
  auto emit = [&](int col, int bin, int alive) {
    const unsigned am = __ballot_sync(FULL, alive != 0);
    int rank = 0;
    unsigned mm = am;
    while (mm) {
      const int src = __ffs(mm) - 1;
      mm &= mm - 1;
      const int b = __shfl_sync(FULL, bin, src);
      rank += (b < bin) ? 1 : 0;
    }
    if (alive) a.pk_bin[(base + col) * maxpks + rank] = (uint8_t)bin;
    const int c = __popc(am);
    if (lane == 0) a.pk_cnt[base + col] = (uint8_t)c;
    if (c) scols = max(scols, col + 1);
    npeaks += c;
  };
  // prefetch ring over columns T-1, T-2, ...: count + this lane's slot (if lane < maxpks)
  int pc[PFB], pb[PFB];
  double pv[PFB];
  const bool slot = lane < maxpks;
  auto fetch = [&](int t, int& c, double& v, int& b) {
    c = a.fwd_cnt[base + t];
    v = slot ? a.fwd_val[(base + t) * maxpks + lane] : 0.0;    // stale beyond the count, never used
    b = slot ? (int)a.fwd_bin[(base + t) * maxpks + lane] : -1;
  };
#pragma unroll
  for (int u = 0; u < PFB; ++u)
    if (T - 1 - u >= 0) fetch(T - 1 - u, pc[u], pv[u], pb[u]);
  for (int t0 = T - 1; t0 >= 0; t0 -= PFB) {
#pragma unroll
    for (int u = 0; u < PFB; ++u) {
      const int t = t0 - u;
      if (t >= 0) {   // warp-uniform
        const int n = pc[u];
        const double my_val = pv[u];
        const int my_bin = (lane < n) ? pb[u] : -1;
        if (t - PFB >= 0) fetch(t - PFB, pc[u], pv[u], pb[u]);
        int cur_alive = 0;
        for (int k = 0; k < n; ++k) {   // stored order is already (value desc, bin desc) (:241)
          const double val = __shfl_sync(FULL, my_val, k);
          const int pos = __shfl_sync(FULL, my_bin, k);
          const bool ok = val >= pick(thr, reg_of(pos));
          if ((__ballot_sync(FULL, ok) >> lane_of(pos)) & 1u) {   // :242, decided by the owning lane
            bump(thr, sE, lane, pos, val);                     // :244-245
            if (lane == k) cur_alive = 1;
            if (nxt_alive && nxt_bin == pos) nxt_alive = 0;    // :247-248 same bin, following column
          }                                                    // else :251 the peak is dropped
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) thr[j] = __dmul_rn(a_dec, thr[j]);
        if (t + 1 < T) emit(t + 1, nxt_bin, nxt_alive);
        nxt_bin = my_bin;
        nxt_alive = cur_alive;
      }
    }
  }
  emit(0, nxt_bin, nxt_alive);
  if (lane == 0) {
    a.item_scols[item] = scols;
    a.item_npeaks[item] = npeaks;
  }
}

// Per-file compaction of one shift's peaks into (col, bin) rows.
__global__ void __launch_bounds__(256) afp_peaks_compact_kernel(const ItemDesc* items, int shifts, int shift,
                                                                int maxpks, const uint8_t* pk_bin,
                                                                const uint8_t* pk_cnt, const int64_t* off,
                                                                int32_t* rows) {
  __shared__ int s_scan[256];
  __shared__ int s_run;
  const ItemDesc it = items[blockIdx.x * shifts + shift];
  const int tid = threadIdx.x;
  if (tid == 0) s_run = 0;
  __syncthreads();
  int32_t* out = rows + 2 * off[blockIdx.x];
  for (int t0 = 0; t0 < it.nframes; t0 += 256) {
    const int t = t0 + tid;
    const int c = (t < it.nframes) ? pk_cnt[it.frame_base + t] : 0;
    s_scan[tid] = c;
    __syncthreads();
    for (int o = 1; o < 256; o <<= 1) {
      const int v = (tid >= o) ? s_scan[tid - o] : 0;
      __syncthreads();
      s_scan[tid] += v;
      __syncthreads();
    }
    const int excl = s_scan[tid] - c + s_run;
    for (int i = 0; i < c; ++i) {
      out[2 * (excl + i)] = t;
      out[2 * (excl + i) + 1] = pk_bin[(it.frame_base + t) * maxpks + i];
    }
    __syncthreads();
    if (tid == 255) s_run += s_scan[255];
    __syncthreads();
  }
}

__global__ void afp_gather_npeaks_kernel(const int32_t* item_npeaks, int nfiles, int shifts, int shift,
                                         int32_t* out) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < nfiles) out[f] = item_npeaks[f * shifts + shift];
}

// Analyzer.spreadpeaksinvector / spreadpeaks as a stand-alone call (audfprint_analyze.py:153-197):
// one CTA; the local maxima of `vec` are listed in shared memory, then every output element
// takes the max over their scaled Gaussians (same products, same max as the reference).
__global__ void __launch_bounds__(256) afp_spread_kernel(const double* vec, int n, const double* tab,
                                                        const double* base, double* out) {
  extern __shared__ int s_pk[];      // indices of the local maxima
  __shared__ int s_n;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const bool ge = (i == 0) ? true : (vec[i] >= vec[i - 1]);          // locmax :46-48
    const bool ge_next = (i == n - 1) ? false : (vec[i + 1] >= vec[i]);
    if (ge && !ge_next) s_pk[atomicAdd(&s_n, 1)] = i;
  }
  __syncthreads();
  const int np = s_n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double v = base ? base[i] : 0.0;
    for (int k = 0; k < np; ++k) {
      const int p = s_pk[k];
      v = fmax(v, __dmul_rn(vec[p], tab[i + n - p]));                  // :195-196
    }
    out[i] = v;
  }
}

}  // namespace

int afp_spread_peaks_impl(afp_ctx* c, const double* vector, int32_t n, const double* table, double width,
                          const double* base, double* out) {
  const size_t nn = (size_t)n;
  AFP_CUDA(c, c->d_tmp.reserve(sizeof(double) * (5 * nn + 8)));
  double* d_vec = c->d_tmp.as<double>();
  double* d_tab = d_vec + nn;             // 2n+1
  double* d_base = d_tab + 2 * nn + 1;
  double* d_out = d_base + nn;
  std::vector<double> tab(2 * nn + 1);
  for (size_t j = 0; j < tab.size(); ++j) {
    const double u = ((double)j - (double)n) / width;
    tab[j] = table ? table[j] : exp(-0.5 * (u * u));
  }
  AFP_CUDA(c, cudaMemcpyAsync(d_vec, vector, sizeof(double) * nn, cudaMemcpyHostToDevice, c->stream));
  AFP_CUDA(c, cudaMemcpyAsync(d_tab, tab.data(), sizeof(double) * tab.size(), cudaMemcpyHostToDevice, c->stream));
  if (base) AFP_CUDA(c, cudaMemcpyAsync(d_base, base, sizeof(double) * nn, cudaMemcpyHostToDevice, c->stream));
  const size_t smem = sizeof(int) * nn;
  if (smem > 48 * 1024)
    AFP_CUDA(c, cudaFuncSetAttribute(afp_spread_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  afp_spread_kernel<<<1, 256, smem, c->stream>>>(d_vec, n, d_tab, base ? d_base : nullptr, d_out);
  AFP_CUDA(c, cudaGetLastError());
  c->launches++;
  AFP_CUDA(c, cudaMemcpyAsync(out, d_out, sizeof(double) * nn, cudaMemcpyDeviceToHost, c->stream));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));   // `tab` must outlive the copy
  return AFP_OK;
}

int afp_launch_peaks(afp_ctx* c, int item0, int nitems) {
  if (nitems <= 0) return AFP_OK;
  PeakArgs a;
  a.items = c->d_items.as<ItemDesc>();
  a.stats = c->d_item_stats.as<ItemStats>();
  a.item0 = item0;
  a.logs = c->d_logs.p;
  a.gauss = c->d_gauss.as<double>();
  a.a_dec = c->ap.a_dec;
  a.pole = c->ap.hpf_pole;
  a.maxpks = c->ap.maxpksperframe;
  a.fwd_val = c->d_fwd_val.as<double>();
  a.fwd_bin = c->d_fwd_bin.as<uint8_t>();
  a.fwd_cnt = c->d_fwd_cnt.as<uint8_t>();
  a.pk_bin = c->d_pk_bin.as<uint8_t>();
  a.pk_cnt = c->d_pk_cnt.as<uint8_t>();
  a.item_scols = c->d_item_scols.as<int32_t>();
  a.item_npeaks = c->d_item_npeaks.as<int32_t>();
  if (!c->peaks_carveout_set) {
    // the whole per-SM shared memory for K2, so that K2_CTAS_PER_SM items fit on every SM
    AFP_CUDA(c, cudaFuncSetAttribute(afp_peaks_kernel<double>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                     cudaSharedmemCarveoutMaxShared));
    AFP_CUDA(c, cudaFuncSetAttribute(afp_peaks_kernel<float>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                     cudaSharedmemCarveoutMaxShared));
    c->peaks_carveout_set = true;
  }
  if (c->ap.spectrogram_fp32) afp_peaks_kernel<float><<<nitems, 32, 0, c->stream>>>(a);
  else afp_peaks_kernel<double><<<nitems, 32, 0, c->stream>>>(a);
  AFP_CUDA(c, cudaGetLastError());
  c->launches++;
  return AFP_OK;
}

int afp_compact_peaks(afp_ctx* c, int shift) {
  // per-file counts of this shift -> offsets -> rows
  AFP_CUDA(c, c->d_tmp.reserve(sizeof(int32_t) * (size_t)(c->nfiles + 1)));
  AFP_CUDA(c, c->d_pk_off.reserve(sizeof(int64_t) * (size_t)(c->nfiles + 1)));
  afp_gather_npeaks_kernel<<<(c->nfiles + 255) / 256, 256, 0, c->stream>>>(
      c->d_item_npeaks.as<int32_t>(), c->nfiles, c->ap.shifts, shift, c->d_tmp.as<int32_t>());
  AFP_CUDA(c, cudaGetLastError());
  c->launches++;
  int rc = afp_launch_scan_i32_to_i64(c, c->d_tmp.as<int32_t>(), c->d_pk_off.as<int64_t>(), c->nfiles);
  if (rc) return rc;
  int64_t total = 0;
  AFP_CUDA(c, cudaMemcpyAsync(&total, c->d_pk_off.as<int64_t>() + c->nfiles, sizeof(int64_t),
                              cudaMemcpyDeviceToHost, c->stream));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  AFP_CUDA(c, c->d_pk_rows.reserve(sizeof(int32_t) * 2 * (size_t)(total + 1)));
  if (total > 0) {
    afp_peaks_compact_kernel<<<c->nfiles, 256, 0, c->stream>>>(
        c->d_items.as<ItemDesc>(), c->ap.shifts, shift, c->ap.maxpksperframe, c->d_pk_bin.as<uint8_t>(),
        c->d_pk_cnt.as<uint8_t>(), c->d_pk_off.as<int64_t>(), c->d_pk_rows.as<int32_t>());
    AFP_CUDA(c, cudaGetLastError());
    c->launches++;
  }
  return AFP_OK;
}
