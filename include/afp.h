/*
 * afp.h — C ABI of libafp.so, the sm_90a (H100) landmark-fingerprint engine.
 *
 * This is the drop-in boundary for the ONE hot path SURVEY.md §8 scopes.  The
 * reference (dpwe/audfprint @ cb03ba99) is pure Python and has no FFI of its
 * own; the "operator API" a replacement must honour is the method set of its
 * three domain classes (SURVEY.md §8b).  Each entry point below names the
 * reference method(s) it stands behind.  The Python mirror of those classes
 * (audfprint_b200/{analyzer,hash_table,matcher}.py) reaches these symbols
 * through ctypes; INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions
 *   - every function returns an int status: 0 = ok, negative = afp_status;
 *     afp_last_error() gives the message.  No exception crosses the ABI.
 *   - plain pointers and sizes only.  A pointer argument named *_dev / with an
 *     `on_host` flag of 0 is a DEVICE pointer (e.g. torch.Tensor.data_ptr());
 *     with on_host = 1 it is a HOST pointer and the library does the
 *     host<->device copy itself on its stream.
 *   - buffers are caller-owned; the context owns only its internal workspace.
 *   - one context per process per GPU; calls are asynchronous on the context's
 *     stream except where a result count must be returned to the host.
 *   - there is no CPU fallback: every call needs a CUDA device.
 */
#ifndef AFP_H_
#define AFP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AFP_ABI_VERSION 2

typedef struct afp_ctx afp_ctx;

typedef enum {
  AFP_OK = 0,
  AFP_ERR_CUDA = -1,        /* a CUDA runtime call failed                       */
  AFP_ERR_INVALID = -2,     /* bad argument (maps to ValueError)               */
  AFP_ERR_UNSUPPORTED = -3, /* parameter outside the compiled limits           */
  AFP_ERR_NOMEM = -4,       /* device workspace allocation failed              */
  AFP_ERR_STATE = -5        /* call order violated (e.g. fetch before compute) */
} afp_status;

enum { AFP_PCM_I16 = 0, AFP_PCM_F32 = 1 };

/* compiled limits */
#define AFP_N_FFT 512
#define AFP_N_HOP 256
#define AFP_NBINS 256           /* bins kept (Nyquist row dropped)           */
#define AFP_MAX_PKS 16          /* maxpksperframe upper bound                */
#define AFP_MAX_MERGE 256       /* shifts*maxpksperframe*maxpairsperpeak cap */

/* Analyzer attributes (audfprint_analyze.py:125-151; set by the CLI at
 * audfprint.py:285-298). */
typedef struct {
  double a_dec;            /* decay per frame, audfprint_analyze.py:277          */
  double hpf_pole;         /* HPF_POLE, audfprint_analyze.py:60                  */
  int32_t maxpksperframe;  /* Analyzer.maxpksperframe (5)                        */
  int32_t maxpairsperpeak; /* Analyzer.maxpairsperpeak (3, --fanout)             */
  int32_t targetdf;        /* 31                                                 */
  int32_t mindt;           /* 2                                                  */
  int32_t targetdt;        /* 63                                                 */
  int32_t shifts;          /* Analyzer.shifts (1; 4 for match)                   */
  int32_t spectrogram_fp32; /* 0 (default): FP64 STFT/log, results bit-identical to the
                             * reference.  1: opt-in FP32 STFT + log + float spectrogram
                             * (K1 at HBM speed; magnitudes within 1e-5 relative, hashes
                             * NOT guaranteed identical - a few files per thousand differ) */
} afp_analyzer_params;

/* Matcher attributes (audfprint_match.py:96-122). */
typedef struct {
  int32_t window;                /* Matcher.window                    */
  int32_t threshcount;           /* Matcher.threshcount               */
  int32_t search_depth;          /* Matcher.search_depth              */
  int32_t max_alignments_per_id; /* Matcher.max_alignments_per_id     */
  int32_t publish_candidates;    /* table-shard mode (SURVEY.md §8e): 0 = off.  1 = rank and report
                                  * the shard's full local top-search_depth ids of every query so
                                  * that one all-gather + afp_fetch_match_candidates can rebuild
                                  * the single-table result (audfprint_b200/dist.py)            */
  int32_t row_capacity;          /* result rows kept per query (0 = 256).  The reference can emit up
                                  * to search_depth * (max_alignments_per_id + 1); a query that
                                  * produces more than this returns AFP_ERR_UNSUPPORTED and the
                                  * caller retries with a larger capacity                       */
  int32_t force_general;         /* 0 = the fast kernel takes every query inside its capacities and
                                  * hands the rest to the general kernel (identical results);
                                  * 1 = general kernel only (tests, A/B timing)                  */
} afp_matcher_params;

/* ---- context --------------------------------------------------------------- */
int afp_abi_version(void);
int afp_create(afp_ctx** out, int device);
void afp_destroy(afp_ctx* ctx);
const char* afp_last_error(afp_ctx* ctx);
/* Use the caller's CUDA stream (cudaStream_t as void*); NULL = library-owned. */
int afp_set_stream(afp_ctx* ctx, void* cuda_stream);
int afp_sync(afp_ctx* ctx);
/* Number of kernel launches issued by this context so far (bench accounting). */
int64_t afp_launch_count(afp_ctx* ctx);

/* Stage timing of afp_fingerprint_batch with CUDA events on the context's stream
 * (bench.py's live roofline measurement).  Stages: 0 host->device PCM copy,
 * 1 K1 stft+log, 2 per-item statistics, 3 K2 peaks, 4 K3 landmarks/merge/write.
 * afp_get_stage_ms synchronises and returns the last batch's durations. */
#define AFP_NSTAGES 5
int afp_set_profiling(afp_ctx* ctx, int enable);
int afp_get_stage_ms(afp_ctx* ctx, float* ms /* [AFP_NSTAGES] */);

/* ---- PCM front-end -----------------------------------------------------------
 * What the reference delegates to `ffmpeg -ac 1 -ar <sr>` plus its reader's scaling
 * (audio_read.py:56-145, :196-203): interleaved int16 PCM of `channels` channels ->
 * mono float32 in [-1, 1) resampled by up/down with the polyphase FIR `taps`
 * (2*half+1 doubles, already scaled by `up`; the host designs them as
 * scipy.signal.resample_poly does).  up = down = 1: down-mix only (taps may be NULL).
 * *nout = ceil(nframes*up/down) samples are written to `out` (HOST or DEVICE float32).
 * Tolerance-pinned, not bit-pinned: no two resamplers agree bit for bit (SURVEY.md 8f-2). */
int afp_pcm_frontend(afp_ctx* ctx, const int16_t* pcm, int pcm_on_host, int64_t nframes, int32_t channels,
                     int32_t up, int32_t down, const double* taps, int32_t ntaps, float* out, int out_on_host,
                     int64_t* nout);

/* ---- Analyzer --------------------------------------------------------------
 * Replaces stft.stft (stft.py:62-94) + Analyzer.find_peaks
 * (audfprint_analyze.py:255-308) + peaks2landmarks (:310-343) +
 * landmarks2hashes (:81-96) + the shift/dedupe logic of wavfile2hashes
 * (:401-422).
 *
 * `window` is the 512-point analysis window (np.hanning(514)[1:-1]) and
 * `gauss` the 513-point spreading table exp(-0.5*((j-256)/f_sd)^2)
 * (audfprint_analyze.py:187-192), both computed by the host so that they are
 * the very doubles the reference multiplies by.  Either may be NULL, in which
 * case the library computes it with libm for f_sd. */
int afp_set_analyzer(afp_ctx* ctx, const afp_analyzer_params* p,
                     const double* window, const double* gauss, double f_sd);

/* Fingerprint a batch of files held as one packed PCM buffer.
 *   pcm            packed samples of all files (int16 or float32)
 *   sample_offsets HOST array [nfiles+1]; file i starts at pcm[off[i]]
 *   sample_lengths HOST array [nfiles] or NULL; NULL means off[i+1]-off[i].
 *                  Explicit lengths let the caller pad each file to a 16-byte
 *                  boundary, which is what lets K1 stage interior tiles with
 *                  TMA bulk copies (unaligned files take the scalar-load path).
 * On return the hashes of every file are in the context workspace;
 * *total_hashes (may be NULL -> no host sync) receives their number. */
int afp_fingerprint_batch(afp_ctx* ctx, const void* pcm, int pcm_dtype, int pcm_on_host,
                          int32_t nfiles, const int64_t* sample_offsets,
                          const int64_t* sample_lengths, int64_t* total_hashes);
/* Copy the result of the last afp_fingerprint_batch: `rows` int32 [total][2]
 * = (time, hash) sorted by (time, hash) per file (audfprint_analyze.py:415-421),
 * `row_offsets` HOST int64 [nfiles+1].  Either may be NULL. */
int afp_fetch_hashes(afp_ctx* ctx, int32_t* rows, int rows_on_host, int64_t* row_offsets);
/* Peaks of one shift of the last batch (Analyzer.find_peaks / wavfile2peaks):
 * `rows` int32 [total][2] = (col, bin) column-major, bins ascending
 * (audfprint_analyze.py:303-308); `row_offsets` HOST int64 [nfiles+1].
 * Call with rows = NULL first to obtain the offsets/total. */
int afp_fetch_peaks(afp_ctx* ctx, int32_t shift, int32_t* rows, int rows_on_host,
                    int64_t* row_offsets);

/* Analyzer.peaks2landmarks (audfprint_analyze.py:310-343) on an explicit peak
 * list (e.g. read from a precomputed .afpk file): `peak_rows` int32 [n][2] =
 * (col, bin), column-major with bins ascending.  Result (fetch): int32 [L][4] =
 * (col, bin1, bin2, dt) in the reference's generation order.  Columns may be
 * anywhere in [0, 2^28]; like afp_fingerprint_batch, the pairing does not depend
 * on how far from column 0 the peaks lie.  Invalidates the last fingerprint batch. */
int afp_landmarks_from_peaks(afp_ctx* ctx, const int32_t* peak_rows, int64_t npeaks, int on_host,
                             int64_t* nlandmarks);
int afp_fetch_landmarks(afp_ctx* ctx, int32_t* rows, int rows_on_host);

/* Analyzer.spreadpeaksinvector (audfprint_analyze.py:153-160) over spreadpeaks (:162-197):
 *   out[i] = max(base[i] (0 when base is NULL), max over the local maxima p of `vector`
 *                (locmax, :36-52) of vector[p] * table[i + n - p]),  0 <= i < n
 * `table` holds the 2n+1 Gaussian values exp(-0.5*((j-n)/width)^2), j = 0..2n, computed by the
 * host with the reference's NumPy expression (:187-192) so that they are the very doubles it
 * multiplies by; NULL = computed here with libm for `width`.  All pointers are HOST pointers
 * (a <=256-element call in the reference); the arithmetic runs on the device. */
int afp_spread_peaks(afp_ctx* ctx, const double* vector, int32_t n, const double* table, double width,
                     const double* base, double* out);

/* Exposed for the STFT parity check (north_star: magnitudes within 1e-5):
 * |STFT| of one signal, float64 [T][257] (frame-major), T = 1 + n/256.
 * Replaces np.abs(stft.stft(d, 512, 256, window)) (audfprint_analyze.py:280). */
int afp_stft_mag(afp_ctx* ctx, const void* pcm, int pcm_dtype, int pcm_on_host, int64_t n,
                 double* mag, int mag_on_host);
/* Conditioned spectrogram log/mean/HPF of one signal, float64 [T][256]
 * (audfprint_analyze.py:280-295). */
int afp_sgram(afp_ctx* ctx, const void* pcm, int pcm_dtype, int pcm_on_host, int64_t n,
              double* sgram, int sgram_on_host);
/* Exposed for the K2/K3 checks: run the product's K2 -> K3 -> merge chain on a caller-supplied
 * log-magnitude spectrogram instead of K1's output.
 *   logs         [sum of item frames][256], double (float in the FP32 spectrogram mode), items
 *                file-major (item f*shifts + s), the same layout as the workspace's d_logs
 *   item_frames  HOST int32 [nfiles*shifts]; an item of shift s > 0 may not be longer than shift 0
 *   item_stats   HOST double [nitems][3] = (logfloor, mean, allzero != 0)
 * Afterwards afp_fetch_hashes / afp_fetch_peaks return results as after afp_fingerprint_batch. */
int afp_fingerprint_from_logs(afp_ctx* ctx, const void* logs, int logs_on_host, int32_t nfiles,
                              const int32_t* item_frames, const double* item_stats, int64_t* total_hashes);

/* ---- HashTable --------------------------------------------------------------
 * Device-resident copy of HashTable.table / counts / hashesperid
 * (hash_table.py:59-81).  `table` uint32 [2^hashbits][depth] row-major,
 * `counts` int32 [2^hashbits], `hashesperid` uint32 [nids]. */
int afp_table_upload(afp_ctx* ctx, const uint32_t* table, const int32_t* counts,
                     int32_t hashbits, int32_t depth, int32_t maxtimebits,
                     const uint32_t* hashesperid, int64_t nids, int on_host);
/* An empty device table (HashTable.__init__ / reset, hash_table.py:59-89). */
int afp_table_create(afp_ctx* ctx, int32_t hashbits, int32_t depth, int32_t maxtimebits);
/* Replace the device copy of hashesperid (host bookkeeping after store / remove). */
int afp_table_set_hashesperid(afp_ctx* ctx, const uint32_t* hashesperid, int64_t nids);
/* HashTable.store (hash_table.py:91-138) for a batch of tracks, on the device table:
 *   rows         int32 [M][2] (time, hash), the files' rows one after the other; NULL = the
 *                hashes of the last afp_fingerprint_batch, taken from the workspace in place
 *   row_offsets  HOST int64 [nfiles+1] (ignored with rows = NULL)
 *   ids          HOST int64 [nfiles] track id of every file (HashTable.name_to_id)
 * Entries that land below `depth` are written (same slots as the reference's sequential loop);
 * entries that hit a full bucket are NOT applied: *noverflow of them wait, in sequence order,
 * for afp_table_fetch_overflow -> (bucket, count before the insert, value).  The reference draws
 * random.randint(0, count) for each of those and writes slot < depth (hash_table.py:127-134): the
 * caller replays the draws (afp_mt_randint_replay) and returns the writes with
 * afp_table_apply_patches (later patches of one slot win, as in the sequential loop: the caller
 * passes one patch per slot). */
int afp_table_store_batch(afp_ctx* ctx, const int32_t* rows, int rows_on_host, const int64_t* row_offsets,
                          int32_t nfiles, const int64_t* ids, int64_t* noverflow);
int afp_table_fetch_overflow(afp_ctx* ctx, uint32_t* bucket, int32_t* count_before, uint32_t* value);
int afp_table_apply_patches(afp_ctx* ctx, const uint32_t* bucket, const int32_t* slot, const uint32_t* value,
                            int64_t n);
/* The same exchange with less traffic (what HashTable.store_batch uses): only the counts travel to
 * the host (the RNG replay needs nothing else), one drawn slot per overflow entry comes back (HOST
 * int32 [noverflow], sequence order; a slot >= depth writes nothing), and the device applies them
 * itself, the LAST entry of a slot winning as in the reference's sequential loop. */
int afp_table_fetch_overflow_counts(afp_ctx* ctx, int32_t* count_before);
int afp_table_apply_slots(afp_ctx* ctx, const int32_t* slot, int64_t n);
/* Copy the device table back: table uint32 [2^hashbits][depth], counts int32 [2^hashbits] (HOST). */
int afp_table_download(afp_ctx* ctx, uint32_t* table, int32_t* counts);
/* CPython's `random.randint(0, count)` replayed for n draws.  state625 = the 625 uint32 of
 * random.getstate()[1] (MT19937 words + position), updated in place so that
 * random.setstate() continues where the reference would.  Host arithmetic only: this is the
 * reference's RNG, not part of the hot path. */
int afp_mt_randint_replay(uint32_t* state625, const int32_t* count_before, int64_t n, int32_t* slot_out);
/* HashTable.remove (hash_table.py:346-364) for n distinct ids in one pass over the device table;
 * removed (HOST [n] or NULL) receives the entries each id had in the table.  A bucket holding an
 * entry of one of the ids keeps its other entries below min(count, depth) in slot order, zeroes the
 * rest of its row and takes their number as its count; other buckets are not written.  The ids'
 * hashesperid become 0.  AFP_ERR_INVALID for an id outside [0, nids) or an id given twice.
 * Not while a store batch is pending: its overflow entries name slots of the table as it was, so
 * finish it (afp_table_apply_slots / afp_table_apply_patches) first. */
int afp_table_remove_ids(afp_ctx* ctx, const int64_t* ids, int64_t n, int64_t* removed);
/* HashTable.retrieve (hash_table.py:366-383) for n ids (repeats allowed): (time, hash) rows of the
 * entries below min(count, depth), hash then slot order, one block per id in request order.
 * *total_rows receives their number; afp_fetch_retrieved copies them, int32 [total][2], and the
 * HOST int64 [n+1] offsets of every id's block. */
int afp_table_retrieve_ids(afp_ctx* ctx, const int64_t* ids, int64_t n, int64_t* total_rows);
int afp_fetch_retrieved(afp_ctx* ctx, int32_t* rows, int rows_on_host, int64_t* row_offsets /* HOST [n+1] */);
/* The fast matching kernel's pruning bound of the device table: its smallest non-zero hashesperid,
 * or 0 (no pruning) when no id has hashes or a live entry names an id whose hashesperid is 0.
 * Recomputed by every call that changes hashesperid (upload, set_hashesperid, remove_ids). */
int afp_table_pruning_bound(afp_ctx* ctx, uint32_t* hmin);
/* Keep only ids in [id_lo, id_hi) of the uploaded table (sharded table,
 * SURVEY.md §8e); bucket-slot order is preserved. */
int afp_table_restrict_ids(afp_ctx* ctx, int64_t id_lo, int64_t id_hi);
/* HashTable.get_hits (hash_table.py:150-176): query rows int32 [nq][2] =
 * (time, hash) -> hits int32 [nhits][4] = (id, dtime, hash, qtime) in
 * (query row, slot) order.  Two steps: count, then fetch. */
int afp_get_hits(afp_ctx* ctx, const int32_t* q_rows, int64_t nq, int q_on_host,
                 int64_t* nhits);
int afp_fetch_hits(afp_ctx* ctx, int32_t* hits, int hits_on_host);

/* ---- Matcher ----------------------------------------------------------------
 * Matcher.match_hashes (audfprint_match.py:314-352) for a batch of queries:
 * get_hits -> _best_count_ids (:124-147) -> _approx_match_counts (:241-312).
 *   q_rows     int32 [sum nq][2] (time, hash) of all queries, packed
 *   q_offsets  HOST int64 [nqueries+1]
 * Result rows int32 [R][7] = (id, count, dtime, raw, rank, 0, 0) per query in
 * candidate-rank order; the final sort by count (:335) is left to the host
 * mirror so that it is the very numpy call the reference makes. */
int afp_match_batch(afp_ctx* ctx, const int32_t* q_rows, int q_on_host, int32_t nqueries,
                    const int64_t* q_offsets, const afp_matcher_params* p,
                    int64_t* total_rows);
int afp_fetch_match_rows(afp_ctx* ctx, int32_t* rows, int rows_on_host, int64_t* row_offsets);
/* afp_match_batch sends a query of rows * depth >= 2^24 to the long-query path (grid-wide passes,
 * memory sized by the query's actual hits, identical rows) unless force_general is set.
 * How many queries of the last afp_match_batch went through the general kernel (all of them
 * with force_general; otherwise the ones outside the fast kernel's capacities, never the long
 * ones). */
int afp_match_general_count(afp_ctx* ctx, int64_t* n);
/* Per query of the last batch, HOST int32 [nqueries][8]:
 *   [0] 0 = the fast kernel finished it, > 0 = why it was handed to the general kernel
 *       (1 multi-record id set full, 2 member-hit list full, 3 too many single-record ids outrank
 *       the K-th member, 4 shard mode with > 2^20 ids and fewer members than search_depth,
 *       5 candidate depth > 1024), 6 = the long-query path finished it (columns 1-7 are 0 then),
 *       -1 = the fast kernel did not run;
 *   [1] multi-record ids, [2] their hits, [3] single-record ids admitted by pass 3,
 *   [4] candidate depth, [5] ids above threshcount, [6] largest bucket multiplicity, [7] distinct
 *       ids (shard mode only). */
int afp_fetch_match_status(afp_ctx* ctx, int32_t* status);
/* After afp_match_batch with publish_candidates = 1: `cand` float64
 * [nqueries][search_depth][3] = (id, raw count, weighted count) in (weight desc, id desc)
 * order, `counts` int32 [nqueries][2] = (entries used, #ids with raw > threshcount). */
int afp_fetch_match_candidates(afp_ctx* ctx, double* cand, int32_t* counts, int on_host);

/* ---- table sharded by track-id range (SURVEY.md 8e; BASELINE configs[4]) -----------------
 * The reference has no such mode; the nearest thing is one table per worker process merged
 * afterwards (audfprint.py:199-235, hash_table.py:291-323).  Every rank uploads the table,
 * keeps its id range (afp_table_restrict_ids), runs afp_match_batch with publish_candidates = 1
 * on ALL queries, packs one fixed-size record per query into a caller-owned DEVICE buffer, the
 * caller all-gathers the buffers (NCCL), and afp_shard_merge rebuilds on the device the rows a
 * single table would give (same rows, same ranks); fetch them with afp_fetch_match_rows.
 * Record (little endian): int32 {n_above, ncand, nrows, 0}; f64 weight[sd]; uint32 id[sd];
 * uint32 raw[sd]; int32 rows[row_cap][7].  row_cap must be even. */
int64_t afp_shard_record_bytes(int32_t search_depth, int32_t row_cap);
int afp_shard_pack(afp_ctx* ctx, int32_t row_cap, void* records_dev /* [nqueries][record bytes] */);
int afp_shard_merge(afp_ctx* ctx, const void* gathered_dev /* [nshards][nqueries][record bytes] */,
                    int32_t nshards, int32_t nqueries, int32_t search_depth, int32_t row_cap,
                    int64_t* total_rows);

#ifdef __cplusplus
}
#endif
#endif /* AFP_H_ */
