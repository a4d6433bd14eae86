// Internal declarations shared by the libafp translation units (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include <string>
#include <utility>
#include <vector>

#include "afp.h"

#define AFP_FRAMES_PER_TILE 16      // frames one CTA pass of K1 transforms
#define AFP_GAUSS_N (2 * AFP_NBINS + 1)
#define AFP_GAUSS_PAD (AFP_GAUSS_N + AFP_GAUSS_N / 8 + 2)   // padded smem layout, see afp_peaks.cu
#define AFP_NO_HASH 0xFFFFFFFFu

// A device buffer that only ever grows (workspace arena member); it owns its allocation.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    std::swap(p, o.p);
    std::swap(cap, o.cap);
    return *this;
  }
  ~DevBuf() {
    if (p) cudaFree(p);
  }
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

// Which allocation of a DevBuf some content was written to: a buffer that grows is reallocated with a
// larger capacity, so (pointer, capacity) names one allocation even if the pointer is reused.
struct BufTag {
  const void* p = nullptr;
  size_t cap = 0;
  bool is(const DevBuf& b) const { return p != nullptr && p == b.p && cap == b.cap; }
  void set(const DevBuf& b) { p = b.p; cap = b.cap; }
  void clear() { p = nullptr; cap = 0; }
};

// Per-item (file x shift) descriptor built on the host for each batch.
struct ItemDesc {
  int64_t sample_start;   // index of the item's first sample in the packed PCM buffer
  int64_t nsamples;       // samples of the item (file length minus the shift offset; may be <= 0)
  int64_t frame_base;     // first frame of the item in the batch-wide frame space
  int32_t nframes;        // T = 1 + nsamples / 256 (0 when nsamples <= 0)
  int32_t tile_base;      // first K1 tile of the item
};

// Per-item statistics produced by K1 + the stats kernel.
struct ItemStats {
  double logfloor;   // log(max|S| / 1e6)
  double mean;       // mean of the floored log-magnitudes over 257 x T
  int32_t allzero;   // 1 when max|S| == 0 (reference skips log/mean, audfprint_analyze.py:287-290)
  int32_t floored;   // 1 while the tile sums of this item still have to be recomputed with the floor
};

struct TableDev {
  DevBuf table, counts, hashesperid;
  int32_t hashbits = 0, depth = 0, maxtimebits = 0;
  int64_t nids = 0;
  uint32_t hmin = 0;   // smallest hashesperid (fast-path pruning bound); 0 = unknown
  bool loaded = false;
};

struct afp_ctx {
  int device = 0;
  int num_sms = 132;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  std::string err;
  int64_t launches = 0;
  bool profiling = false;
  cudaEvent_t ev[AFP_NSTAGES + 1] = {};
  bool ev_valid = false;
  // host->device pipelining of afp_fingerprint_batch (pcm_on_host)
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_chunk[32] = {};
  cudaEvent_t ev_batch_done = nullptr;
  cudaStream_t chunk_stream[4] = {};   // chunks are processed round-robin on these
  cudaEvent_t ev_chunk_stream[4] = {};

  // analyzer configuration
  afp_analyzer_params ap{};
  bool analyzer_set = false;
  bool peaks_carveout_set = false;   // K2's shared-memory carveout has been raised on this device
  DevBuf d_window;   // 2 x 512 doubles: window, then window * 2^-15 (int16 PCM)
  DevBuf d_gauss;    // AFP_GAUSS_N doubles
  DevBuf d_window_f; // float copies for the FP32 spectrogram mode
  DevBuf d_twid_f;   // float2: tw256[p][r] (256), W512^k (256)
  DevBuf d_twid;     // double2 tables: tw256[p][r] (256), W512^k (256), log table (64 entries x 8 copies)

  // batch state (valid after afp_fingerprint_batch)
  int32_t nfiles = 0, nitems = 0;
  int64_t total_frames = 0, total_tiles = 0, total_cols = 0;
  std::vector<ItemDesc> h_items;
  std::vector<int64_t> h_file_col_base;   // [nfiles+1] column space of each file (= T of shift 0)
  bool batch_valid = false;
  int pcm_dtype = 0;

  // What d_items / d_file_col_base hold (uploaded by reserve_batch) and whether d_tile_item was built from
  // them: a batch with the same layout as the last one skips both uploads and the tile table.  Code that
  // writes these buffers otherwise clears the tags.
  std::vector<ItemDesc> up_items;
  std::vector<int64_t> up_file_col_base;
  BufTag items_tag, fcb_tag, tile_tag;

  DevBuf d_pcm_stage;      // host->device staging when pcm_on_host
  DevBuf d_items;          // ItemDesc[nitems]
  DevBuf d_tile_item;      // int32[total_tiles] item of every K1 tile
  DevBuf d_file_col_base;  // int64[nfiles+1]
  DevBuf d_logs;           // double [total_frames][256]   log|S|, bins 0..255
  DevBuf d_nyq;            // double [total_frames]        log|S| of the Nyquist bin
  DevBuf d_tile_stats;     // double [total_tiles][3]      (max |S|^2, min log, sum log)
  DevBuf d_item_stats;     // ItemStats[nitems]
  DevBuf d_stats_ticket;   // int32 [nitems]  CTAs of an item that finished its floored tile sums
  DevBuf d_fwd_val;        // double [total_frames][maxpks]
  DevBuf d_fwd_bin;        // uint8  [total_frames][maxpks]
  DevBuf d_fwd_cnt;        // uint8  [total_frames]
  DevBuf d_pk_bin;         // uint8  [total_frames][maxpks]  surviving peaks, bins ascending
  DevBuf d_pk_cnt;         // uint8  [total_frames]
  DevBuf d_item_scols;     // int32 [nitems]  last peak column + 1
  DevBuf d_item_npeaks;    // int32 [nitems]
  DevBuf d_lm;             // uint32 [frames][maxpks][fanout] landmark hashes (AFP_NO_HASH = none), afp_landmarks_from_peaks
  DevBuf d_col_cnt;        // int32 [frames]       landmarks per column; then exclusive offsets, afp_landmarks_from_peaks
  DevBuf d_file_tot;       // int32 [nfiles]       rows of each file
  DevBuf d_file_off;       // int64 [nfiles+1]
  DevBuf d_hash_stage;     // int32 [maxpks*fanout*total_frames][2]  K3's rows, file by file at maxpks*fanout*frame_base
  DevBuf d_hashes;         // int32 [total][2]
  int64_t total_hashes = -1;
  int64_t nlandmarks = -1;   // afp_landmarks_from_peaks result (rows in d_hashes)
  DevBuf d_pk_off;         // int64 [nfiles+1] (peak fetch)
  DevBuf d_pk_rows;        // int32 [total][2]
  DevBuf d_pk_in;          // int32 [rows][2]  host peak rows staged for afp_fingerprint_from_peaks / afp_landmarks_from_peaks
  DevBuf d_pk_inoff;       // int64 [nfiles+1] their per-file offsets
  DevBuf d_pk_status;      // int32 [nfiles]   per-file PK_* flags of the peak scatter (afp_hash.cu)
  DevBuf d_tmp;            // misc
  DevBuf d_cub;            // CUB's temporary storage (cub_call)

  // table + matching
  TableDev tab;
  DevBuf d_q, d_qoff, d_hit_off, d_hits;
  int64_t nhits = -1, hits_nq = 0;
  // device-side HashTable.store (afp_store.cu)
  DevBuf d_st_off, d_st_ids, d_st_eval, d_st_seq, d_st_ovf, d_st_cnt, d_st_seg, d_st_heavy, d_st_part, d_st_scan;
  DevBuf d_st_obkt, d_st_opos, d_st_oval, d_st_slot, d_st_last;
  int64_t store_novf = 0;
  // device-side HashTable.remove / retrieve for a list of ids (afp_table_edit.cu)
  DevBuf d_ed_ids, d_ed_bits, d_ed_slot, d_ed_cnt, d_ed_off, d_ed_key, d_ed_key2, d_ed_val, d_ed_val2;
  DevBuf d_ed_uoff, d_ed_req, d_ed_rows;
  int64_t rt_total = -1;              // rows of the last afp_table_retrieve_ids; -1 = none
  int rt_src = 0;                     // where they are: 0 d_ed_val, 1 d_ed_val2, 2 d_ed_rows
  std::vector<int64_t> h_rt_off;      // [n+1] row offsets per requested id
  // device-side HashTable.merge (afp_table_merge.cu): incoming rows + counts, per-bucket flags and
  // pool sizes, their scan, overflowing buckets + pool sizes, one chunk's pool indices and new rows
  DevBuf d_mg_in, d_mg_flag, d_mg_off, d_mg_bkt, d_mg_idx, d_mg_row;
  DevBuf d_mfast, d_mqlist;    // fast path: member-hit lists; [count + pad][query list] handed to the general kernel
  int64_t match_general = 0;   // queries of the last batch the general kernel processed
  int match_general_h = 0;
  bool match_fast_ran = false;
  DevBuf d_mscratch, d_mrows, d_mrow_cnt, d_mrow_off, d_mrows_packed, d_mcand, d_mcand_cnt;
  int32_t match_sdepth = 0;
  bool match_published = false;
  int32_t match_nq = 0;
  int64_t match_total_rows = -1;
  int32_t match_row_cap = 0;
  uint64_t match_layout = 0;   // carve-up of d_mscratch whose counters/histograms are known to be zero
  // long-query path (afp_match_long.cu): sort keys, per-id counters and slots, ranking
  // keys, candidate segments and rows, candidates' hits, per-CTA dtime histograms
  DevBuf d_lg_key, d_lg_id, d_lg_w, d_lg_cand, d_lg_dts, d_lg_hist;
  int lg_ctas = 0;                  // CTAs of the mode pass (one histogram pair each)
  std::vector<int> match_long;      // queries of the last batch the long-query path finished
  // exact_count / find_time_range finish (afp_match_options.cu): per-slot segments and lookup,
  // routed hits, approximate-row flags, mode supports, packed keys, qtimes, finished rows
  DevBuf d_op_slot, d_op_hit, d_op_mode, d_op_sup, d_op_key, d_op_tq, d_op_rows;
  // the same finish on one shard of an id-range sharded table, in two calls around the caller's
  // all-reduce of the per-query largest qtime: what the ranking call leaves for the finish call,
  // and the smallest local rank per query whose quantile read failed (0x7f7f7f7f: none)
  struct {
    bool pending = false;        // afp_match_options_shard_rank ran; its finish has not
    bool finished = false;       // the last result is a shard finish: afp_shard_pack packs it
    afp_matcher_params p{};
    int32_t nq = 0, exact = 0, trange = 0;
    int64_t nrows = 0, ranked = 0;
    double quant = 0.0;
    int64_t breaks[32] = {};
    const int32_t* dq = nullptr;
  } sopt;
  DevBuf d_op_qfail;
  // FLAC decoding (afp_flac.cu): staged compressed bytes, per-byte header candidates, file descriptors,
  // per-file locate results, the frame tables and the int32 samples before decorrelation
  DevBuf d_fl_in, d_fl_cand, d_fl_file, d_fl_res, d_fl_frame, d_fl_scratch;
  struct {
    bool valid = false;              // afp_flac_locate_batch ran and its batch has not been decoded over
    int32_t nfiles = 0;
    const uint8_t* bytes = nullptr;  // device bytes the frame table points into
    std::vector<int64_t> nsamples;   // per file, per channel (0 for a failed file)
    std::vector<int32_t> nframes, status;
    std::vector<char> desc;          // the FlacFile descriptors of the batch
  } fl;
};

#define AFP_CUDA(ctx, call)                                                        \
  do {                                                                             \
    cudaError_t e__ = (call);                                                      \
    if (e__ != cudaSuccess) {                                                      \
      (ctx)->err = std::string(#call) + ": " + cudaGetErrorString(e__);            \
      return (e__ == cudaErrorMemoryAllocation) ? AFP_ERR_NOMEM : AFP_ERR_CUDA;    \
    }                                                                              \
  } while (0)

#define AFP_FAIL(ctx, code, msg) \
  do {                           \
    (ctx)->err = (msg);          \
    return (code);               \
  } while (0)

// ---- launches, copies and scratch: every entry point goes through these -----------------------

// Launch `kernel` on c->stream as it is now (run_chunked switches it per chunk) and count one launch
// in afp_launch_count.  An empty grid is no launch.  Above 48 KB of dynamic shared memory the kernel's
// limit is raised first.
template <class... P, class... A>
int afp_launch(afp_ctx* c, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A&&... args) {
  if ((size_t)grid.x * grid.y * grid.z == 0) return AFP_OK;
  if (smem > 48 * 1024)
    AFP_CUDA(c, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<grid, block, smem, c->stream>>>(std::forward<A>(args)...);
  AFP_CUDA(c, cudaGetLastError());
  c->launches++;
  return AFP_OK;
}

// A two-phase CUB call f(temp, bytes): the size query, then the call with the context's temporary
// buffer.  Counts one launch, whatever CUB runs.
template <class F>
int cub_call(afp_ctx* c, F f) {
  size_t bytes = 0;
  AFP_CUDA(c, f(nullptr, bytes));
  AFP_CUDA(c, c->d_cub.reserve(bytes + 16));
  AFP_CUDA(c, f(c->d_cub.p, bytes));
  c->launches++;
  return AFP_OK;
}

// n values of the device array src to dst, which is host memory or device memory as dst_on_host says;
// queued on c->stream.
template <class T>
cudaError_t afp_copy_out(afp_ctx* c, T* dst, const T* src, size_t n, int dst_on_host) {
  return cudaMemcpyAsync(dst, src, sizeof(T) * n, dst_on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice,
                         c->stream);
}

// n values of the caller's array src, host memory or device memory as src_on_host says, to the device
// array dst; queued on c->stream.
template <class T>
cudaError_t afp_copy_in(afp_ctx* c, T* dst, const T* src, size_t n, int src_on_host) {
  return cudaMemcpyAsync(dst, src, sizeof(T) * n, src_on_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice,
                         c->stream);
}

// The caller's n values of T on the device: *dev = src itself when it is device memory, else its copy in
// `stage` (queued on c->stream).
template <class T>
int afp_stage(afp_ctx* c, DevBuf& stage, const T* src, size_t n, int on_host, const T** dev) {
  *dev = src;
  if (!on_host || n == 0) return AFP_OK;
  AFP_CUDA(c, stage.reserve(sizeof(T) * n + 16));
  AFP_CUDA(c, afp_copy_in(c, stage.as<T>(), src, n, 1));
  *dev = stage.as<T>();
  return AFP_OK;
}

inline cudaError_t afp_read_async(afp_ctx*) { return cudaSuccess; }
template <class T, class... R>
cudaError_t afp_read_async(afp_ctx* c, T* h, const T* d, size_t n, R... rest) {
  const cudaError_t e = cudaMemcpyAsync(h, d, sizeof(T) * n, cudaMemcpyDeviceToHost, c->stream);
  return e != cudaSuccess ? e : afp_read_async(c, rest...);
}

// Host copies of device values behind everything queued on c->stream, and one synchronise for all of
// them: afp_read_back(c, &x, d_x, 1, v.data(), d_v, n, ...).
template <class... A>
int afp_read_back(afp_ctx* c, A... a) {
  AFP_CUDA(c, afp_read_async(c, a...));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  return AFP_OK;
}

// Consecutive 16-byte-aligned arrays of one DevBuf.  afp_carve runs the same take<T>(n) sequence twice:
// a Carver without a base only adds up the bytes to reserve, then one on the buffer hands out the arrays.
struct Carver {
  char* base = nullptr;
  size_t bytes = 0;   // offset of the next array
  template <class T> T* take(int64_t n) {
    T* r = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
    bytes += ((size_t)std::max<int64_t>(n, 1) * sizeof(T) + 15) & ~(size_t)15;
    return r;
  }
};

template <class F>
int afp_carve(afp_ctx* c, DevBuf& buf, F layout) {
  Carver size;
  layout(size);
  AFP_CUDA(c, buf.reserve(size.bytes));
  Carver arrays{buf.as<char>()};
  layout(arrays);
  return AFP_OK;
}

// What a workspace buffer may grow to: half of the free device memory plus what `held` holds already,
// and at least 1 GiB.
inline cudaError_t afp_memory_budget(const DevBuf& held, size_t* budget) {
  size_t free_b = 0, total_b = 0;
  const cudaError_t e = cudaMemGetInfo(&free_b, &total_b);
  *budget = std::max<size_t>((free_b + held.cap) / 2, (size_t)1 << 30);
  return e;
}

// ---- kernel launchers (defined in the .cu files) -------------------------------
int afp_launch_tile_table(afp_ctx* c);
int afp_launch_stft(afp_ctx* c, const void* pcm, int dtype, double* mag_out /* optional [T][257] */, int64_t tile0,
                    int64_t ntiles);
int afp_launch_stats(afp_ctx* c, int item0, int nitems);
int afp_launch_sgram(afp_ctx* c, double* sgram_out);
int afp_launch_peaks(afp_ctx* c, int item0, int nitems);
int afp_launch_file_hashes(afp_ctx* c, int file0, int nfiles);   // K3 of files file0 .. file0+nfiles-1, to d_hash_stage
int afp_launch_hashes(afp_ctx* c);   // file row counts -> d_file_off (all files)
int afp_write_hashes(afp_ctx* c);    // d_hash_stage -> dense d_hashes
int afp_landmarks_from_peaks_impl(afp_ctx* c, const int32_t* rows, int64_t n, int on_host, int64_t* nlm);
// peak rows of a ragged batch -> pk_bin / pk_cnt at each file's item (items f * item_stride of d_items)
int afp_launch_scatter_peaks(afp_ctx* c, const int32_t* rows, const int64_t* off, int64_t nrows, int32_t nfiles,
                             int item_stride, int32_t* status);
int afp_launch_peak_last_cols(afp_ctx* c, const int32_t* rows, const int64_t* off, int32_t nfiles, int32_t* out);
int afp_peak_status_code(int32_t bits);   // a file's scatter flags -> AFP_OK / AFP_ERR_INVALID / AFP_ERR_UNSUPPORTED
int afp_compact_peaks(afp_ctx* c, int shift);
int afp_spread_peaks_impl(afp_ctx* c, const double* vector, int32_t n, const double* table, double width,
                          const double* base, double* out);
int afp_launch_scan_i32_to_i64(afp_ctx* c, const int32_t* in, int64_t* out, int64_t n);
extern "C" int afp_table_stats(afp_ctx* c);
int afp_finish_match_rows(afp_ctx* c, int nqueries, int row_cap, int64_t* total_out);
int afp_scan_large(afp_ctx* c, const int32_t* in, int64_t* out, int64_t n);   // afp_store.cu
