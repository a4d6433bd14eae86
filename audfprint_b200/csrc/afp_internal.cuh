// Internal declarations shared by the libafp translation units (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>

#include "afp.h"

#define AFP_FRAMES_PER_TILE 16      // frames one CTA pass of K1 transforms
#define AFP_GAUSS_N (2 * AFP_NBINS + 1)
#define AFP_GAUSS_PAD (AFP_GAUSS_N + AFP_GAUSS_N / 8 + 2)   // padded smem layout, see afp_peaks.cu
#define AFP_NO_HASH 0xFFFFFFFFu

// A device buffer that only ever grows (workspace arena member).
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
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
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
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

  DevBuf d_pcm_stage;      // host->device staging when pcm_on_host
  DevBuf d_items;          // ItemDesc[nitems]
  DevBuf d_tile_item;      // int32[total_tiles] item of every K1 tile
  DevBuf d_file_col_base;  // int64[nfiles+1]
  DevBuf d_logs;           // double [total_frames][256]   log|S|, bins 0..255
  DevBuf d_nyq;            // double [total_frames]        log|S| of the Nyquist bin
  DevBuf d_tile_stats;     // double [total_tiles][3]      (max |S|^2, min log, sum log)
  DevBuf d_item_stats;     // ItemStats[nitems]
  DevBuf d_fwd_val;        // double [total_frames][maxpks]
  DevBuf d_fwd_bin;        // uint8  [total_frames][maxpks]
  DevBuf d_fwd_cnt;        // uint8  [total_frames]
  DevBuf d_pk_bin;         // uint8  [total_frames][maxpks]  surviving peaks, bins ascending
  DevBuf d_pk_cnt;         // uint8  [total_frames]
  DevBuf d_item_scols;     // int32 [nitems]  last peak column + 1
  DevBuf d_item_npeaks;    // int32 [nitems]
  DevBuf d_lm;             // uint32 [total_frames][maxpks][fanout] landmark hashes (AFP_NO_HASH = none)
  DevBuf d_col_cnt;        // int32 [total_cols]   unique hashes per (file, column); then exclusive offsets
  DevBuf d_file_tot;       // int32 [nfiles]
  DevBuf d_file_off;       // int64 [nfiles+1]
  DevBuf d_hashes;         // int32 [total][2]
  int64_t total_hashes = -1;
  int64_t nlandmarks = -1;   // afp_landmarks_from_peaks result (rows in d_hashes)
  DevBuf d_pk_off;         // int64 [nfiles+1] (peak fetch)
  DevBuf d_pk_rows;        // int32 [total][2]
  DevBuf d_tmp;            // misc

  // table + matching
  TableDev tab;
  DevBuf d_q, d_qoff, d_hit_off, d_hits;
  int64_t nhits = -1, hits_nq = 0;
  // device-side HashTable.store (afp_store.cu)
  DevBuf d_st_off, d_st_ids, d_st_eval, d_st_seq, d_st_ovf, d_st_cnt, d_st_seg, d_st_heavy, d_st_part, d_st_scan;
  DevBuf d_st_obkt, d_st_opos, d_st_oval, d_st_slot, d_st_last;
  int64_t store_novf = 0;
  // device-side HashTable.remove / retrieve for a list of ids (afp_table_edit.cu)
  DevBuf d_ed_ids, d_ed_bits, d_ed_slot, d_ed_cnt, d_ed_off, d_ed_key, d_ed_key2, d_ed_val, d_ed_val2, d_ed_cub;
  DevBuf d_ed_uoff, d_ed_req, d_ed_rows;
  int64_t rt_total = -1;              // rows of the last afp_table_retrieve_ids; -1 = none
  int rt_src = 0;                     // where they are: 0 d_ed_val, 1 d_ed_val2, 2 d_ed_rows
  std::vector<int64_t> h_rt_off;      // [n+1] row offsets per requested id
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
  // long-query path (afp_match_long.cu): sort keys, CUB temp, per-id counters and slots, ranking
  // keys, candidate segments and rows, candidates' hits, per-CTA dtime histograms
  DevBuf d_lg_key, d_lg_cub, d_lg_id, d_lg_w, d_lg_cand, d_lg_dts, d_lg_hist;
  int lg_ctas = 0;                  // CTAs of the mode pass (one histogram pair each)
  std::vector<int> match_long;      // queries of the last batch the long-query path finished
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

// ---- kernel launchers (defined in the .cu files) -------------------------------
int afp_launch_tile_table(afp_ctx* c);
int afp_launch_stft(afp_ctx* c, const void* pcm, int dtype, double* mag_out /* optional [T][257] */, int64_t tile0,
                    int64_t ntiles);
int afp_launch_stats(afp_ctx* c, int item0, int nitems);
int afp_launch_sgram(afp_ctx* c, double* sgram_out);
int afp_launch_peaks(afp_ctx* c, int item0, int nitems);
int afp_launch_landmarks(afp_ctx* c, int item0, int nitems);
int afp_launch_hashes(afp_ctx* c);   // merge / scans (all files)
int afp_write_hashes(afp_ctx* c);
int afp_landmarks_from_peaks_impl(afp_ctx* c, const int32_t* rows, int64_t n, int on_host, int64_t* nlm);
int afp_compact_peaks(afp_ctx* c, int shift);
int afp_spread_peaks_impl(afp_ctx* c, const double* vector, int32_t n, const double* table, double width,
                          const double* base, double* out);
int afp_launch_scan_i32_to_i64(afp_ctx* c, const int32_t* in, int64_t* out, int64_t n);
extern "C" int afp_table_stats(afp_ctx* c);
int afp_finish_match_rows(afp_ctx* c, int nqueries, int row_cap, int64_t* total_out);
int afp_scan_large(afp_ctx* c, const int32_t* in, int64_t* out, int64_t n);   // afp_store.cu
