// K3 — peak-pair fan-out, 20-bit hash packing, cross-shift merge/sort/dedupe.
//
// Replaces Analyzer.peaks2landmarks (audfprint_analyze.py:310-343),
// landmarks2hashes (:81-96) and the concatenate / sort / unique tail of
// wavfile2hashes (:401-422).
//
// Layout trick: every (item, column) owns maxpks fixed peak slots (bins
// ascending) and every peak owns `fanout` hash slots, so no prefix sums are
// needed until the very end.  All hashes of one file that carry the same time
// value live in the same column of its (up to `shifts`) items; the final
// (time, hash)-sorted, de-duplicated output of a file is therefore the
// concatenation over columns of the sorted unique union of at most
// shifts*maxpks*fanout slot values — a per-thread insertion sort.
#include "afp_internal.cuh"

namespace {

struct HashArgs {
  const ItemDesc* items;
  int file0;                    // first file of the launch
  int shifts, maxpks, fanout, targetdf, mindt, targetdt;
  int win;                      // source columns per window
  const uint8_t* pk_bin;
  const uint8_t* pk_cnt;
  const int32_t* item_scols;
  uint32_t* lm;                 // [frames][maxpks][fanout]      (afp_landmarks_from_peaks)
  const int64_t* file_col_base; // [nfiles+1]                    (afp_landmarks_from_peaks)
  int32_t* col_cnt;             // [cols] counts, then offsets   (afp_landmarks_from_peaks)
  int32_t* file_tot;            // [nfiles] rows of each file
  const int64_t* file_off;      // [nfiles+1]
  int32_t* stage;               // [P*F*frames][2] file f's rows from row P*F*(frame_base of its shift-0 item)
  int32_t* hashes;              // [total][2]
};

constexpr int K3_THREADS = 256;

// Exclusive prefix of v over the CTA's K3_THREADS threads in thread order; *total gets the sum.
// s_w holds K3_THREADS / 32 ints.
__device__ __forceinline__ int block_excl_scan(int v, int* s_w, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_w[w] = x;
  __syncthreads();
  int before = 0, tot = 0;
#pragma unroll
  for (int k = 0; k < K3_THREADS / 32; ++k) {
    const int t = s_w[k];
    before += (k < w) ? t : 0;
    tot += t;
  }
  *total = tot;
  __syncthreads();   // s_w is rewritten by the next call
  return before + x - v;
}

// The peaks of a window of S items, compacted into shared memory in the order the reference visits
// them: item by item, each sorted by (column, bin).  Item s (last peak column + 1 s_scols[s], first
// frame s_fb[s], both in shared memory so that a column's count is the only dependent load) contributes
// its columns [w0, min(s_scols[s], w0 + span)); its entries are s_pk[s_seg[s] .. s_seg[s+1]), packed
// (col - w0):20 | slot:4 | bin:8.  The column is stored relative to the window start, so a window of
// any item's length fits the 20-bit field.  Ends with a barrier.
__device__ __forceinline__ void compact_window(const HashArgs& a, const int* s_scols, const int64_t* s_fb, int S,
                                               int w0, int span, uint32_t* s_pk, int* s_seg, int* s_w) {
  const int P = a.maxpks;
  int run = 0;
  for (int j0 = 0; j0 < S * span; j0 += K3_THREADS) {
    const int j = j0 + threadIdx.x;
    const int s = j / span, c = w0 + (j - s * span);
    int n = 0;
    int64_t fc = 0;
    if (j < S * span && c < s_scols[s]) {
      fc = s_fb[s] + c;
      n = a.pk_cnt[fc];
    }
    int tot;
    const int at = run + block_excl_scan(n, s_w, &tot);
    if (j < S * span && c == w0) s_seg[s] = at;
    for (int k = 0; k < n; ++k) s_pk[at + k] = ((uint32_t)(c - w0) << 12) | ((uint32_t)k << 8) | a.pk_bin[fc * P + k];
    run += tot;
  }
  if (threadIdx.x == 0) s_seg[S] = run;
  __syncthreads();
}

// The hashes of source entry i of one item's window list s_pk[.. end) (column < scols): its pairs with
// the entries that follow it, in (column, bin) order, at most `fanout` (audfprint_analyze.py:325-343),
// packed as landmarks2hashes packs them (:92-95).  Returns how many were written to out.
__device__ __forceinline__ int pair_source(const HashArgs& a, const uint32_t* s_pk, int i, int end, int w0, int scols,
                                           uint32_t* out) {
  const uint32_t e = s_pk[i];
  const int col = w0 + (int)(e >> 12), slot = (int)((e >> 8) & 15), b1 = (int)(e & 255);
  const int c2lo = col + a.mindt, c2hi = min(scols, col + a.targetdt);     // :331-332
  int n = 0;
  for (int j = (a.mindt > 0) ? i + 1 : i - slot; j < end && n < a.fanout; ++j) {
    const uint32_t t = s_pk[j];
    const int c2 = w0 + (int)(t >> 12);
    if (c2 >= c2hi) break;
    if (c2 < c2lo) continue;
    const int b2 = (int)(t & 255);
    if (abs(b2 - b1) < a.targetdf)                                          // :335
      out[n++] = ((uint32_t)(b1 & 0xFF) << 12) | ((uint32_t)((b2 - b1) & 0x3F) << 6) | (uint32_t)((c2 - col) & 0x3F);
  }
  return n;
}

// Landmarks of one item (afp_landmarks_from_peaks): every peak owns `fanout` slots of lm, pre-filled
// with AFP_NO_HASH by a memset.  One thread per source peak.
constexpr int PCAP = 11264;   // peak entries per window
static_assert(PCAP <= (1 << 20), "a window's relative column must fit the 20-bit field");

__global__ void __launch_bounds__(K3_THREADS) afp_landmark_kernel(HashArgs a) {
  __shared__ uint32_t s_pk[PCAP];
  __shared__ int s_seg[2];
  __shared__ int s_w[K3_THREADS / 32];
  __shared__ int s_scols[1];
  __shared__ int64_t s_fb[1];
  const int scols = a.item_scols[0];                       // last peak column + 1 (:321)
  const int P = a.maxpks, F = a.fanout;
  const int64_t base = a.items[0].frame_base;
  const int W = max(64, PCAP / P - a.targetdt - 1);       // source columns per window: P * (W + targetdt) <= PCAP
  if (threadIdx.x == 0) {
    s_scols[0] = scols;
    s_fb[0] = base;
  }
  __syncthreads();
  for (int w0 = 0; w0 < scols; w0 += W) {
    compact_window(a, s_scols, s_fb, 1, w0, W + a.targetdt, s_pk, s_seg, s_w);
    const int np = s_seg[1];
    for (int i = threadIdx.x; i < np; i += K3_THREADS) {
      const uint32_t e = s_pk[i];
      const int col = w0 + (int)(e >> 12);
      if (col >= w0 + W) break;                           // entries are column-sorted: only targets remain
      pair_source(a, s_pk, i, np, w0, scols, a.lm + ((base + col) * P + ((e >> 8) & 15)) * F);
    }
    __syncthreads();
  }
}

// K3 of the fingerprint batch: one CTA per file, window by window over its columns.  The peaks of the
// file's `shifts` items are compacted (compact_window) and paired into hash slots in shared memory,
// [column][shift][slot][fanout] (AFP_NO_HASH = empty).  All hashes of a file that carry the same time
// value live in one column, so its (time, hash)-sorted unique rows (the concatenate / sort / unique
// tail of wavfile2hashes, :401-422) are, column by column, the sorted unique union of that column's
// slots: an insertion sort in place, one thread per column.  The rows go to the file's staging region,
// whose P*F slots per frame of all its items bound its row count; file_tot gets the count.
constexpr int K3_SLOTS = 4096;   // hash slots of a window: W * shifts * maxpks * fanout <= K3_SLOTS

// 8 CTAs per SM (32 registers, no spills; 27 KB of shared memory each at the default settings, with the
// carveout at its maximum): a batch of 1024 files is one wave on 132 SMs
__global__ void __launch_bounds__(K3_THREADS, 8) afp_file_hash_kernel(HashArgs a) {
  extern __shared__ uint32_t s_pk[];          // shifts * maxpks * (W + targetdt) entries
  __shared__ uint32_t s_slot[K3_SLOTS];
  __shared__ int s_seg[AFP_MAX_MERGE + 1];
  __shared__ int s_w[K3_THREADS / 32];
  __shared__ int s_scols[AFP_MAX_MERGE];     // shifts <= AFP_MAX_MERGE
  __shared__ int64_t s_fb[AFP_MAX_MERGE];
  const int f = a.file0 + blockIdx.x, S = a.shifts, it0 = f * S, tid = threadIdx.x;
  const int P = a.maxpks, F = a.fanout, SPF = S * P * F, W = a.win;
  for (int s = tid; s < S; s += K3_THREADS) {
    s_scols[s] = a.item_scols[it0 + s];
    s_fb[s] = a.items[it0 + s].frame_base;
  }
  __syncthreads();
  int scols = 0;
  for (int s = 0; s < S; ++s) scols = max(scols, s_scols[s]);
  int2* out = reinterpret_cast<int2*>(a.stage) + (int64_t)P * F * s_fb[0];
  int run = 0;
  for (int w0 = 0; w0 < scols; w0 += W) {
    const int ncol = min(W, scols - w0);
    for (int e = tid; e < ncol * SPF; e += K3_THREADS) s_slot[e] = AFP_NO_HASH;
    compact_window(a, s_scols, s_fb, S, w0, W + a.targetdt, s_pk, s_seg, s_w);
    for (int s = 0; s < S; ++s) {
      const int end = s_seg[s + 1], sc = s_scols[s];
      for (int i = s_seg[s] + tid; i < end; i += K3_THREADS) {
        const uint32_t e = s_pk[i];
        const int cc = (int)(e >> 12);
        if (cc >= W) break;                       // entries are column-sorted: only targets remain
        pair_source(a, s_pk, i, end, w0, sc, s_slot + ((cc * S + s) * P + (int)((e >> 8) & 15)) * F);
      }
    }
    __syncthreads();
    for (int c0 = 0; c0 < ncol; c0 += K3_THREADS) {
      const int cc = c0 + tid;
      uint32_t* buf = s_slot + cc * SPF;
      int n = 0;
      if (cc < ncol)
        for (int e = 0; e < SPF; ++e) {           // reads slot e, writes slots < n <= e
          const uint32_t h = buf[e];
          if (h == AFP_NO_HASH) continue;
          int i = n;
          while (i > 0 && buf[i - 1] > h) --i;
          if (i > 0 && buf[i - 1] == h) continue; // duplicate across shifts (:417)
          for (int k = n; k > i; --k) buf[k] = buf[k - 1];
          buf[i] = h;
          ++n;
        }
      int tot;
      const int at = run + block_excl_scan(n, s_w, &tot);
      for (int k = 0; k < n; ++k) out[at + k] = make_int2(w0 + cc, (int)buf[k]);
      run += tot;
    }
    __syncthreads();                              // s_slot and s_pk are refilled by the next window
  }
  if (tid == 0) a.file_tot[f] = run;
}

// Each file's rows from its staging region to their place in the dense output.
__global__ void __launch_bounds__(256) afp_gather_rows_kernel(HashArgs a) {
  const int f = blockIdx.x;
  const int64_t n = a.file_off[f + 1] - a.file_off[f];
  const int2* src = reinterpret_cast<const int2*>(a.stage) +
                    (int64_t)a.maxpks * a.fanout * a.items[(int64_t)f * a.shifts].frame_base;
  int2* dst = reinterpret_cast<int2*>(a.hashes) + a.file_off[f];
  for (int64_t i = threadIdx.x; i < n; i += 256) dst[i] = src[i];
}

// In-place exclusive scan of col_cnt inside each file; file totals out.
__global__ void __launch_bounds__(256) afp_file_scan_kernel(HashArgs a) {
  __shared__ int s_scan[256];
  __shared__ int s_run;
  const int f = blockIdx.x, tid = threadIdx.x;
  const int64_t c0 = a.file_col_base[f];
  const int ncol = (int)(a.file_col_base[f + 1] - c0);
  if (tid == 0) s_run = 0;
  __syncthreads();
  for (int t0 = 0; t0 < ncol; t0 += 256) {
    const int t = t0 + tid;
    const int c = (t < ncol) ? a.col_cnt[c0 + t] : 0;
    s_scan[tid] = c;
    __syncthreads();
    for (int o = 1; o < 256; o <<= 1) {
      const int v = (tid >= o) ? s_scan[tid - o] : 0;
      __syncthreads();
      s_scan[tid] += v;
      __syncthreads();
    }
    if (t < ncol) a.col_cnt[c0 + t] = s_scan[tid] - c + s_run;
    __syncthreads();
    if (tid == 255) s_run += s_scan[255];
    __syncthreads();
  }
  if (tid == 0) a.file_tot[f] = s_run;
}

// Single-CTA exclusive scan int32[n] -> int64[n+1].
__global__ void __launch_bounds__(1024) afp_scan_kernel(const int32_t* in, int64_t* out, int64_t n) {
  __shared__ long long s_scan[1024];
  __shared__ long long s_run;
  const int tid = threadIdx.x;
  if (tid == 0) s_run = 0;
  __syncthreads();
  for (int64_t i0 = 0; i0 < n; i0 += 1024) {
    const int64_t i = i0 + tid;
    const long long c = (i < n) ? in[i] : 0;
    s_scan[tid] = c;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      const long long v = (tid >= o) ? s_scan[tid - o] : 0;
      __syncthreads();
      s_scan[tid] += v;
      __syncthreads();
    }
    if (i < n) out[i] = s_scan[tid] - c + s_run;
    __syncthreads();
    if (tid == 1023) s_run += s_scan[1023];
    __syncthreads();
  }
  if (tid == 0) out[n] = s_run;
}

// ---- explicit peak lists -> K2's output layout (peaks2landmarks / .afpk hashing as calls) ----
// One thread per peak row of a ragged batch: rows[off[f] .. off[f+1]) are file f's (col, bin) pairs,
// rows indexed absolutely (row off[0] is the first).  The row finds its file by binary search over
// `off` (the largest f with off[f] <= row: empty files share their offset with the next file) and
// lands at the file's frame_base + col in pk_bin / pk_cnt, in the slot its rank in the column gives.
// status[f] collects PK_BAD_LAYOUT (a column outside [0, T_f) or a bin outside [0, 256), or rows not
// column-major with bins ascending) and PK_TOO_MANY (more than maxpks peaks in one column); a row that
// sets either writes nothing, so pk_cnt never exceeds maxpks whatever the input.
constexpr int PK_BAD_LAYOUT = 1, PK_TOO_MANY = 2;

__global__ void __launch_bounds__(256) afp_scatter_peaks_kernel(const int32_t* rows, const int64_t* off, int nfiles,
                                                               const ItemDesc* items, int item_stride, int maxpks,
                                                               uint8_t* pk_bin, uint8_t* pk_cnt, int32_t* status) {
  const int64_t i = off[0] + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= off[nfiles]) return;
  int f = 0, hi = nfiles;
  while (hi - f > 1) {
    const int mid = (f + hi) >> 1;
    if (off[mid] <= i) f = mid; else hi = mid;
  }
  const int64_t b = off[f];
  const ItemDesc it = items[(int64_t)f * item_stride];   // nframes = T_f = last peak column + 1
  const int col = rows[2 * i], bin = rows[2 * i + 1];
  if (col < 0 || col >= it.nframes || bin < 0 || bin >= AFP_NBINS ||
      (i > b && (rows[2 * (i - 1)] > col || (rows[2 * (i - 1)] == col && rows[2 * (i - 1) + 1] >= bin)))) {
    atomicOr(&status[f], PK_BAD_LAYOUT);
    return;
  }
  int slot = 0;
  while (i - slot - 1 >= b && rows[2 * (i - slot - 1)] == col) {
    if (++slot >= maxpks) {
      atomicOr(&status[f], PK_TOO_MANY);
      return;
    }
  }
  pk_bin[(it.frame_base + col) * maxpks + slot] = (uint8_t)bin;
  if (i + 1 == off[f + 1] || rows[2 * (i + 1)] != col) pk_cnt[it.frame_base + col] = (uint8_t)(slot + 1);
}

// Column of each non-empty file's last row (-1 for an empty file): its T_f - 1 (:321).
__global__ void afp_peak_last_col_kernel(const int32_t* rows, const int64_t* off, int nfiles, int32_t* out) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < nfiles) out[f] = off[f + 1] > off[f] ? rows[2 * (off[f + 1] - 1)] : -1;
}

template <bool WRITE>
__global__ void afp_lm_rows_kernel(const uint32_t* lm, int T, int PF, int32_t* col_cnt, int32_t* out) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= T) return;
  const uint32_t* src = lm + (int64_t)col * PF;
  int n = 0;
  int32_t* dst = WRITE ? out + 4 * (int64_t)col_cnt[col] : nullptr;
  for (int e = 0; e < PF; ++e) {
    const uint32_t h = src[e];
    if (h == AFP_NO_HASH) continue;
    if (WRITE) {   // inverse packing, audfprint_analyze.py:99-112
      const int b1 = (h >> 12) & 0xFF;
      int df = (h >> 6) & 0x3F;
      if (df >= 32) df -= 64;
      dst[4 * n] = col; dst[4 * n + 1] = b1; dst[4 * n + 2] = b1 + df; dst[4 * n + 3] = h & 0x3F;
    }
    ++n;
  }
  if (!WRITE) col_cnt[col] = n;
}

}  // namespace

static HashArgs make_args(afp_ctx* c) {
  HashArgs a;
  a.items = c->d_items.as<ItemDesc>();
  a.file0 = 0;
  a.shifts = c->ap.shifts;
  a.maxpks = c->ap.maxpksperframe;
  a.fanout = c->ap.maxpairsperpeak;
  a.targetdf = c->ap.targetdf;
  a.mindt = c->ap.mindt;
  a.targetdt = c->ap.targetdt;
  // source columns per window of afp_file_hash_kernel: whole passes of K3_THREADS columns when they fit
  const int w = K3_SLOTS / (a.shifts * a.maxpks * a.fanout);
  a.win = w >= K3_THREADS ? w / K3_THREADS * K3_THREADS : w;
  a.pk_bin = c->d_pk_bin.as<uint8_t>();
  a.pk_cnt = c->d_pk_cnt.as<uint8_t>();
  a.item_scols = c->d_item_scols.as<int32_t>();
  a.lm = c->d_lm.as<uint32_t>();
  a.file_col_base = c->d_file_col_base.as<int64_t>();
  a.col_cnt = c->d_col_cnt.as<int32_t>();
  a.file_tot = c->d_file_tot.as<int32_t>();
  a.file_off = c->d_file_off.as<int64_t>();
  a.stage = c->d_hash_stage.as<int32_t>();
  a.hashes = c->d_hashes.as<int32_t>();
  return a;
}

int afp_peak_status_code(int32_t bits) {
  return (bits & PK_BAD_LAYOUT) ? AFP_ERR_INVALID : (bits & PK_TOO_MANY) ? AFP_ERR_UNSUPPORTED : AFP_OK;
}

int afp_launch_peak_last_cols(afp_ctx* c, const int32_t* rows, const int64_t* off, int32_t nfiles, int32_t* out) {
  return afp_launch(c, afp_peak_last_col_kernel, (nfiles + 255) / 256, 256, 0, rows, off, nfiles, out);
}

int afp_launch_scatter_peaks(afp_ctx* c, const int32_t* rows, const int64_t* off, int64_t nrows, int32_t nfiles,
                             int item_stride, int32_t* status) {
  return afp_launch(c, afp_scatter_peaks_kernel, (unsigned)((nrows + 255) / 256), 256, 0, rows, off, nfiles,
                    c->d_items.as<ItemDesc>(), item_stride, c->ap.maxpksperframe, c->d_pk_bin.as<uint8_t>(),
                    c->d_pk_cnt.as<uint8_t>(), status);
}

int afp_landmarks_from_peaks_impl(afp_ctx* c, const int32_t* rows_in, int64_t n, int on_host, int64_t* nlm) {
  c->batch_valid = false;
  c->nlandmarks = -1;
  if (n == 0) { c->nlandmarks = 0; if (nlm) *nlm = 0; return AFP_OK; }
  const int32_t* drows = nullptr;
  int32_t last[2];
  int rc = afp_stage(c, c->d_pk_in, rows_in, 2 * (size_t)n, on_host, &drows);
  if (rc) return rc;
  if (on_host) last[0] = rows_in[2 * (n - 1)];
  else if ((rc = afp_read_back(c, last, rows_in + 2 * (n - 1), 2))) return rc;
  if (last[0] < 0 || last[0] > (1 << 28)) AFP_FAIL(c, AFP_ERR_INVALID, "bad peak column");
  const int T = last[0] + 1;   // scols = last peak column + 1 (:321)
  const size_t P = (size_t)c->ap.maxpksperframe, F = (size_t)c->ap.maxpairsperpeak, fr = (size_t)T + 1;
  ItemDesc it{};
  it.nframes = T;
  AFP_CUDA(c, c->d_items.reserve(sizeof(ItemDesc) * 2));
  AFP_CUDA(c, c->d_pk_bin.reserve(P * fr));
  AFP_CUDA(c, c->d_pk_cnt.reserve(fr));
  AFP_CUDA(c, c->d_item_scols.reserve(sizeof(int32_t) * 2));
  AFP_CUDA(c, c->d_lm.reserve(sizeof(uint32_t) * P * F * fr));
  AFP_CUDA(c, c->d_col_cnt.reserve(sizeof(int32_t) * fr));
  AFP_CUDA(c, c->d_file_tot.reserve(sizeof(int32_t) * 4));
  AFP_CUDA(c, c->d_file_col_base.reserve(sizeof(int64_t) * 2));
  AFP_CUDA(c, c->d_pk_inoff.reserve(sizeof(int64_t) * 2));
  AFP_CUDA(c, c->d_pk_status.reserve(sizeof(int32_t) * 2));
  const int64_t fcb[2] = {0, T}, off[2] = {0, n};
  c->items_tag.clear();   // written here, not by reserve_batch
  c->fcb_tag.clear();
  c->tile_tag.clear();
  AFP_CUDA(c, cudaMemcpyAsync(c->d_items.p, &it, sizeof(it), cudaMemcpyHostToDevice, c->stream));
  AFP_CUDA(c, cudaMemcpyAsync(c->d_file_col_base.p, fcb, sizeof(fcb), cudaMemcpyHostToDevice, c->stream));
  AFP_CUDA(c, cudaMemcpyAsync(c->d_pk_inoff.p, off, sizeof(off), cudaMemcpyHostToDevice, c->stream));
  AFP_CUDA(c, cudaMemcpyAsync(c->d_item_scols.p, &T, sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
  AFP_CUDA(c, cudaMemsetAsync(c->d_pk_cnt.p, 0, fr, c->stream));
  AFP_CUDA(c, cudaMemsetAsync(c->d_pk_status.p, 0, sizeof(int32_t), c->stream));
  rc = afp_launch_scatter_peaks(c, drows, c->d_pk_inoff.as<int64_t>(), n, 1, 1, c->d_pk_status.as<int32_t>());
  if (rc) return rc;
  c->nfiles = 1; c->nitems = 1; c->total_frames = T; c->total_cols = T;
  HashArgs a = make_args(c);
  AFP_CUDA(c, cudaMemsetAsync(c->d_lm.p, 0xFF, sizeof(uint32_t) * P * F * fr, c->stream));
  int32_t total = 0, err = 0;
  if ((rc = afp_launch(c, afp_landmark_kernel, 1, K3_THREADS, 0, a)) ||
      (rc = afp_launch(c, afp_lm_rows_kernel<false>, (T + 127) / 128, 128, 0, a.lm, T, (int)(P * F), a.col_cnt,
                       nullptr)) ||
      (rc = afp_launch(c, afp_file_scan_kernel, 1, 256, 0, a)) ||
      (rc = afp_read_back(c, &total, c->d_file_tot.as<int32_t>(), 1, &err, c->d_pk_status.as<int32_t>(), 1)))
    return rc;
  if (afp_peak_status_code(err) == AFP_ERR_INVALID)
    AFP_FAIL(c, AFP_ERR_INVALID, "peak rows must be (col, bin) in [0,T)x[0,256), column-major, bins ascending");
  if (err) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "more peaks in one column than maxpksperframe");
  AFP_CUDA(c, c->d_hashes.reserve(sizeof(int32_t) * 4 * (size_t)(total + 1)));
  if (total > 0 &&
      (rc = afp_launch(c, afp_lm_rows_kernel<true>, (T + 127) / 128, 128, 0, a.lm, T, (int)(P * F), a.col_cnt,
                       c->d_hashes.as<int32_t>())))
    return rc;
  c->nlandmarks = total;
  if (nlm) *nlm = total;
  return AFP_OK;
}

int afp_launch_scan_i32_to_i64(afp_ctx* c, const int32_t* in, int64_t* out, int64_t n) {
  return afp_launch(c, afp_scan_kernel, 1, 1024, 0, in, out, n);
}

int afp_launch_file_hashes(afp_ctx* c, int file0, int nfiles) {
  if (nfiles <= 0) return AFP_OK;
  HashArgs a = make_args(c);
  a.file0 = file0;
  const size_t smem = sizeof(uint32_t) * a.shifts * a.maxpks * (a.win + a.targetdt);
  AFP_CUDA(c, cudaFuncSetAttribute(afp_file_hash_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                   cudaSharedmemCarveoutMaxShared));
  return afp_launch(c, afp_file_hash_kernel, nfiles, K3_THREADS, smem, a);
}

int afp_launch_hashes(afp_ctx* c) {
  if (c->nfiles == 0) return AFP_OK;
  return afp_launch_scan_i32_to_i64(c, c->d_file_tot.as<int32_t>(), c->d_file_off.as<int64_t>(), c->nfiles);
}

int afp_write_hashes(afp_ctx* c) {
  if (c->total_cols == 0) return AFP_OK;
  return afp_launch(c, afp_gather_rows_kernel, c->nfiles, 256, 0, make_args(c));
}
