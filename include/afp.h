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
 *   - stream order is the caller's to keep at the boundary.  A device buffer a
 *     call reads must be complete with respect to the context's stream: if other
 *     streams wrote it, make the context's stream wait for them (e.g. an event)
 *     before the call.  A device buffer a call writes must no longer be in use
 *     by work on other streams.  A buffer (device or pinned host) read by a call
 *     that returns without synchronising (afp_fingerprint_batch with
 *     total_hashes = NULL) must stay unchanged and allocated until the next call
 *     that synchronises the context's stream (afp_sync, any fetch).
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
  AFP_ERR_STATE = -5,       /* call order violated (e.g. fetch before compute) */
  AFP_ERR_INDEX = -6        /* a computed index leaves its array (maps to IndexError) */
} afp_status;

/* Sample formats.  afp_fingerprint_batch takes AFP_PCM_I16 and AFP_PCM_F32 (float in [-1, 1)); the
 * byte forms of the front-ends (afp_pcm_frontend_batch_bytes, afp_swr_frontend_batch_bytes) take all
 * four, packed little-endian as a WAV data chunk holds them: int16, IEEE float32, 24-bit integers in 3
 * bytes, 32-bit integers.  A 17-24-bit FLAC file decoded at full depth is AFP_PCM_S32 holding
 * x << (32 - bits). */
enum { AFP_PCM_I16 = 0, AFP_PCM_F32 = 1, AFP_PCM_S24 = 2, AFP_PCM_S32 = 3 };

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
  int32_t window;                /* Matcher.window, 0 .. 4096         */
  int32_t threshcount;           /* Matcher.threshcount, >= 0 (a negative one is AFP_ERR_INVALID:
                                  * the reference's rows there are degenerate, DESIGN.md §8)    */
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
/* Use the caller's CUDA stream (cudaStream_t as void*); NULL = library-owned.  Waits for the work
 * queued on the outgoing stream (the caller's or the library's) first, so that no call on the new
 * stream overtakes it in the shared workspace; the outgoing stream must still exist. */
int afp_set_stream(afp_ctx* ctx, void* cuda_stream);
/* The stream the context's calls run on: the caller's (afp_set_stream) or the library-owned one. */
int afp_get_stream(afp_ctx* ctx, void** cuda_stream);
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
 * Each output is the correctly rounded float32 of
 *   out[n] = sum_j taps[n*down + half - j*up] * RN32(sum_c pcm[j][c] / (32768 channels)),
 * except in a tie zone where the exact sum lies within the float64 accumulation's error bound of a
 * float32 rounding boundary (there: within 1 ulp).  Held to an extended-precision statement of that
 * sum (tests/exact_resample.py), with scipy.signal.resample_poly as its CPU cross-check.  ffmpeg's
 * resampler, which the reference uses, is not reproduced (SURVEY.md 8f-2).
 * AFP_ERR_INVALID for nframes < 0, channels < 1, up or down < 1, a resampling call without an
 * odd-length `taps`, or NULL pcm/out with nframes > 0; nframes = 0 gives *nout = 0. */
int afp_pcm_frontend(afp_ctx* ctx, const int16_t* pcm, int pcm_on_host, int64_t nframes, int32_t channels,
                     int32_t up, int32_t down, const double* taps, int32_t ntaps, float* out, int out_on_host,
                     int64_t* nout);
/* afp_pcm_frontend for a list of files in one launch, every output bit-identical to that file
 * through afp_pcm_frontend alone (both kernels call one per-output function).
 *   pcm            packed interleaved int16 of all files, HOST or DEVICE, pcm_len int16 values
 *   pcm_offsets    HOST int64 [nfiles]: file i's frames start at pcm[pcm_offsets[i]]
 *   nframes, channels, up, down   HOST [nfiles]: file i's frame count, channel count and rate ratio
 *   pair_rates     HOST int32 [npairs][2]: the distinct (up, down) of the resampled files
 *   tap_offsets    HOST int64 [npairs+1], taps HOST float64: pair p's odd-length design (resample_taps)
 *                  is taps[tap_offsets[p] .. tap_offsets[p+1]); each pair is uploaded once per call
 *   out            DEVICE float32 of out_capacity samples, or NULL for a sizing call
 *   out_offsets    HOST int64 [nfiles+1] (may be NULL): file i's ceil(nframes*up/down) outputs start
 *                  at out[out_offsets[i]], a multiple of 4 (16 bytes); out_offsets[nfiles] is the
 *                  buffer length the call needs.  out_lengths HOST int64 [nfiles] (may be NULL).
 * The layout is afp_fingerprint_batch's packed float32 input (sample_offsets = out_offsets,
 * sample_lengths = out_lengths).  Nothing outside each file's [start, start + length) is written.
 * Every argument is checked before anything is launched: AFP_ERR_INVALID for a negative length,
 * channels < 1, up or down < 1, a resampled file whose (up, down) has no taps, an even-length
 * design, an input range outside [0, pcm_len), or an output larger than out_capacity.  One kernel
 * launch and one stream synchronise for the whole list; none when no file has an output. */
int afp_pcm_frontend_batch(afp_ctx* ctx, const int16_t* pcm, int pcm_on_host, int64_t pcm_len, int32_t nfiles,
                           const int64_t* pcm_offsets, const int64_t* nframes, const int32_t* channels,
                           const int32_t* up, const int32_t* down, int32_t npairs, const int32_t* pair_rates,
                           const int64_t* tap_offsets, const double* taps, float* out, int64_t out_capacity,
                           int64_t* out_offsets, int64_t* out_lengths);
/* afp_pcm_frontend_batch over packed payload bytes with a sample format per file:
 *   pcm            pcm_bytes bytes, HOST or DEVICE: each file's samples as its WAV data chunk holds them
 *   byte_offsets   HOST int64 [nfiles]: file i starts at byte byte_offsets[i], a multiple of its sample's
 *                  width for AFP_PCM_I16 (2), AFP_PCM_S32 and AFP_PCM_F32 (4) when counted from an
 *                  aligned address; AFP_PCM_S24 takes any offset
 *   formats        HOST int32 [nfiles]: AFP_PCM_* of each file
 * Each sample enters the down-mix as the int16 `ffmpeg -ac 1` gives a mono file of its format at its own
 * rate: x >> 16 of a 24-bit (x << 8) or 32-bit integer, and for a float v the packed s16 rule of the
 * ffmpeg front-end below.  An all-AFP_PCM_I16 call is afp_pcm_frontend_batch, bit for bit, through the
 * same kernel; files of every format share one launch.  AFP_ERR_INVALID for an unknown format or a
 * misaligned file, otherwise as afp_pcm_frontend_batch. */
int afp_pcm_frontend_batch_bytes(afp_ctx* ctx, const uint8_t* pcm, int pcm_on_host, int64_t pcm_bytes, int32_t nfiles,
                                 const int64_t* byte_offsets, const int32_t* formats, const int64_t* nframes,
                                 const int32_t* channels, const int32_t* up, const int32_t* down, int32_t npairs,
                                 const int32_t* pair_rates, const int64_t* tap_offsets, const double* taps, float* out,
                                 int64_t out_capacity, int64_t* out_offsets, int64_t* out_lengths);

/* ---- ffmpeg front-end (audfprint_b200/csrc/afp_swr.cu) ----
 * What `ffmpeg -i F -f s16le -ac 1 -ar <out_rate> -` (the reference's reader, audio_read.py:196-203)
 * makes of 16-bit mono or stereo PCM, bit for bit, scaled to float32 v / 32768: libswresample's s16
 * down-mix at equal rates, and at other rates its float32 polyphase resampler (Kaiser, beta 9,
 * cut-off 0.97, 32 taps per output period, exact-rational phases) summed in the order of its x86 FMA3
 * kernel, with its edge reflections and output count.  tests/swr_reference.py states it in NumPy.
 *
 * afp_swr_design: the float32 bank of in_rate -> out_rate, host only (no device, no context):
 * *phases = P, *taps = L (either may be NULL) and, when bank is not NULL, P x L floats (row p = phase
 * p) into bank[0 .. capacity).  AFP_ERR_UNSUPPORTED when out / gcd(in, out) > 1024 (a rate such as
 * 44099 Hz needs interpolated phases) or a design longer than 528 taps (above 176400 Hz, not yet
 * matched to the library); AFP_ERR_INVALID for a rate < 1 or a capacity below P L. */
int afp_swr_design(int32_t in_rate, int32_t out_rate, float* bank, int64_t capacity, int32_t* phases, int32_t* taps);
/* afp_swr_length: host only, *nout = the samples afp_swr_frontend_batch gives a mono or stereo file of
 * nframes frames at in_rate (nframes itself at equal rates).  AFP_ERR_UNSUPPORTED for a rate
 * afp_swr_design refuses; AFP_ERR_INVALID for nframes < 0, a rate < 1, NULL nout or a file too long. */
int afp_swr_length(int64_t nframes, int32_t in_rate, int32_t out_rate, int64_t* nout);
/* afp_swr_frontend_batch: the layout and calls of afp_pcm_frontend_batch (a sizing call with out =
 * NULL, then the compute call; pcm HOST or DEVICE; out DEVICE in afp_fingerprint_batch's packed layout),
 * with each file's input rate in `rates` HOST int32 [nfiles] instead of up/down and taps: the library
 * designs each distinct rate once per process and uploads it once per call.  out_lengths are the
 * library's output counts.  AFP_ERR_UNSUPPORTED for more than 2 channels or a rate afp_swr_design
 * refuses; AFP_ERR_INVALID as afp_pcm_frontend_batch.  One launch and one synchronise per call. */
int afp_swr_frontend_batch(afp_ctx* ctx, const int16_t* pcm, int pcm_on_host, int64_t pcm_len, int32_t nfiles,
                           const int64_t* pcm_offsets, const int64_t* nframes, const int32_t* channels,
                           const int32_t* rates, int32_t out_rate, float* out, int64_t out_capacity,
                           int64_t* out_offsets, int64_t* out_lengths);
/* afp_swr_frontend_batch over packed payload bytes with a sample format per file (the layout of
 * afp_pcm_frontend_batch_bytes).  What FFmpeg 8.0 does with 24-bit, 32-bit and float PCM, and with
 * 17-24-bit FLAC decoded at full depth (AFP_PCM_S32, afp_flac_decode_batch_bytes): its decoders give an
 * integer as the int32 x << (32 - bits) and a float as it is, and libswresample then makes int16
 *   mono, equal rates    x >> 16 of an integer; the s16 rule of a float;
 *   stereo, equal rates  in float32: each channel as float(x) 2^-31 (or the float), 0.5 l + 0.5 r, the
 *                        s16 rule;
 *   other rates          the float32 resampler above, fed those floats instead of x / 32768.
 * s16 rule: v * 32768 in float32, rounded half to even to int32, NaN, +-Inf and values outside the int32
 * range giving INT32_MIN, then saturated to int16: so NaN, +Inf and large positive values give -32768
 * (x86 cvtps2dq + packssdw).  The library converts the last n % 16 samples of each buffer with its scalar
 * rule instead, av_clip_int16((int) lrintf(v * 32768)), which differs only for NaN, +-Inf and |v| >= 65536:
 * for float input at equal rates the buffers are 4096-byte packets and the kernel takes the scalar rule
 * for the file's last nframes % 16 outputs; at other rates the packed rule is taken for every output.
 * An all-AFP_PCM_I16 call is afp_swr_frontend_batch, bit for bit, through the same kernel.  8-bit, 64-bit
 * float, A-law, mu-law and other codings have no format code: the library's int16 and double engines they
 * would go through are not stated.  AFP_ERR_INVALID for an unknown format or a misaligned file,
 * otherwise as afp_swr_frontend_batch. */
int afp_swr_frontend_batch_bytes(afp_ctx* ctx, const uint8_t* pcm, int pcm_on_host, int64_t pcm_bytes, int32_t nfiles,
                                 const int64_t* byte_offsets, const int32_t* formats, const int64_t* nframes,
                                 const int32_t* channels, const int32_t* rates, int32_t out_rate, float* out,
                                 int64_t out_capacity, int64_t* out_offsets, int64_t* out_lengths);

/* ---- FLAC decoding -----------------------------------------------------------
 * What the reference's `ffmpeg -i F -f s16le` does for a FLAC file, up to the int16 stream the PCM
 * front-end takes: the frames of a list of FLAC streams are decoded on the device into interleaved
 * int16, in the layout afp_pcm_frontend_batch takes as its device input.  Two calls:
 *   afp_flac_locate_batch  finds every file's frames and returns its sample count (one synchronise);
 *   afp_flac_decode_batch  decodes the located files into a caller-owned DEVICE buffer.
 * The host parses the metadata blocks and passes, per file, the byte range of its frames (everything
 * after the last metadata block) and the STREAMINFO fields below.
 *
 * Locate: every byte that starts a frame header (sync code, no reserved value, fields consistent with
 * STREAMINFO, correct CRC-8) is a candidate.  From the first byte of the file, a frame ends at the next
 * candidate whose frame number (fixed block size) or first-sample number (variable block size; below
 * 2^31, as FFmpeg reads no 7-byte coded number) follows on and where the CRC-16 over [frame start, candidate) is right; the last frame ends at the
 * end of the file's bytes.  So a sync pattern inside compressed data never splits a frame.  STREAMINFO's
 * total sample count is not used (it may be 0): the count is the sum of the frames' block sizes.
 *
 * Decode: CONSTANT, VERBATIM, FIXED (orders 0-4) and LPC (orders 1-32, int64 accumulation)
 * subframes, wasted bits, Rice partitions with 4- and 5-bit parameters and escape partitions,
 * independent, left/side, right/side and mid/side channels, block sizes 1-65535, fixed or variable;
 * 4-24 bits per sample, 1-8 channels.  A b-bit sample x becomes the int16 FFmpeg's decoder and
 * libswresample give: x << (16 - b) for b <= 16, x >> (b - 16) (arithmetic) above.
 * The STREAMINFO MD5 signature is not checked (ffmpeg does not check it by default either).
 *
 * A file is refused, with its own code in file_status, for a depth outside 4-24 bits, a frame chain
 * that does not follow on, a CRC-16 mismatch, a reserved code, a last frame cut short, or subframe data
 * that does not fit its frame.  ffmpeg would conceal a bad frame and go on; here the whole file is
 * refused.  A refused file gets no samples (count 0) and nothing is written for it; nothing outside a
 * file's output range is written.  Both calls return AFP_OK when no file failed, else the code of the
 * lowest failing file: AFP_ERR_UNSUPPORTED for a depth, AFP_ERR_INVALID for the others. */
typedef struct {
  int64_t byte_offset;      /* first byte of the file's frames in the packed bytes */
  int64_t nbytes;           /* bytes of frames (to the end of the file) */
  int32_t sample_rate;      /* STREAMINFO fields */
  int32_t channels;         /* 1-8 */
  int32_t bits_per_sample;  /* 4-24 decodable */
  int32_t max_blocksize;    /* a frame header with a larger block size is not a candidate (if >= 16) */
} afp_flac_stream;

enum {
  AFP_FLAC_OK = 0,
  AFP_FLAC_DEPTH = 1,       /* bits per sample outside 4-24 (25-32 are not decoded) */
  AFP_FLAC_CHAIN = 2,       /* no frame at the start, or a frame followed by one that does not follow on */
  AFP_FLAC_CRC = 3,         /* a frame's CRC-16 does not match */
  AFP_FLAC_RESERVED = 4,    /* a reserved code in a frame or subframe header */
  AFP_FLAC_TRUNCATED = 5,   /* the last frame does not end in its CRC-16 (cut short, or damaged: no
                             * later header tells the two apart) */
  AFP_FLAC_CORRUPT = 6      /* subframe data that does not fit its frame (residual past the frame's
                             * end, a partition order the block size cannot take, a negative LPC shift),
                             * or that FFmpeg's decoder refuses: wasted bits >= the subframe's depth, a
                             * residual of -2^31, a Rice quotient of 2^(32 - k) + 1 or more (2^31 - 1 for
                             * k < 2).  A quotient of exactly 2^(32 - k) is read as FFmpeg reads it: one
                             * more bit b, u = b + 1. */
};

/*   bytes         packed FLAC frame bytes of all files, HOST or DEVICE, nbytes_total of them.  A DEVICE
 *                 buffer is read by both calls and must stay unchanged until afp_flac_decode_batch
 *                 returns.
 *   files         HOST [nfiles]
 *   nsamples      HOST int64 [nfiles] or NULL: samples per channel of every file (0 when it fails)
 *   file_status   HOST int32 [nfiles] or NULL: AFP_FLAC_* of every file */
int afp_flac_locate_batch(afp_ctx* ctx, const uint8_t* bytes, int bytes_on_host, int64_t nbytes_total,
                          int32_t nfiles, const afp_flac_stream* files, int64_t* nsamples, int32_t* file_status);
/* Decode the files of the last afp_flac_locate_batch: file i's nsamples[i] * channels interleaved int16
 * go to out_dev[out_offsets[i] ...] (HOST int64 [nfiles]); out_dev holds out_capacity int16.  Files that
 * failed to locate are skipped.  file_status (HOST [nfiles] or NULL) receives the codes of both calls;
 * a file that fails here may have had part of its own range written.  AFP_ERR_STATE without a located
 * batch; every range is checked against out_capacity before anything is launched.  Synchronises. */
int afp_flac_decode_batch(afp_ctx* ctx, int16_t* out_dev, int64_t out_capacity, const int64_t* out_offsets,
                          int32_t* file_status);
/* afp_flac_decode_batch into a byte buffer: out_dev holds out_capacity bytes and file i starts at byte
 * out_offsets[i].  With full_depth = 0 every file is int16 as above.  With full_depth = 1 a file of 17-24
 * bits is written at full depth, AFP_PCM_S32 holding x << (32 - b) (4 bytes a sample, 4-byte aligned),
 * the int32 FFmpeg's decoder gives it; files of 16 bits or fewer are int16 (2-byte aligned) either way.
 * AFP_ERR_INVALID for a misaligned file; otherwise as afp_flac_decode_batch. */
int afp_flac_decode_batch_bytes(afp_ctx* ctx, uint8_t* out_dev, int64_t out_capacity, const int64_t* out_offsets,
                                int32_t full_depth, int32_t* file_status);

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
/* wavfile2hashes of many precomputed-peak (.afpk) files in one pass (audfprint_analyze.py:385-426:
 * peaks2landmarks, landmarks2hashes, sorted unique (time, hash) rows).
 *   peak_rows     int32 [..][2] (col, bin), column-major with bins ascending per file, HOST or DEVICE
 *   peak_offsets  HOST int64 [nfiles+1], non-decreasing: file f is rows [off[f], off[f+1]) of peak_rows
 *   file_status   HOST int32 [nfiles] or NULL: 0, or the code afp_landmarks_from_peaks returns for that
 *                 file alone (AFP_ERR_INVALID: a column outside [0, 2^28] or past the file's last
 *                 column, a bin outside [0, 256), rows out of order; AFP_ERR_UNSUPPORTED: more peaks
 *                 in one column than maxpksperframe)
 * A file has last column + 1 columns (:321); an empty file has none and no hashes.  The result is
 * left in the workspace exactly as afp_fingerprint_batch leaves it: afp_fetch_hashes,
 * afp_table_store_batch(rows = NULL) and afp_fetch_peaks(shift 0, which returns the input) work on it,
 * at any configured number of shifts.  When a file fails, the call returns the code of the lowest
 * failing file and leaves no batch to fetch or store.  The workspace holds about
 * (maxpksperframe * (1 + 4 maxpairsperpeak) + 5) bytes per column of the batch, plus 8 per hash. */
int afp_fingerprint_from_peaks(afp_ctx* ctx, const int32_t* peak_rows, int rows_on_host, int32_t nfiles,
                               const int64_t* peak_offsets, int32_t* file_status, int64_t* total_hashes);

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
/* HashTable.merge (hash_table.py:291-323) of one incoming table into the device table.
 *   table, counts  HOST uint32 [2^hashbits][depth] and int32 [2^hashbits] of the incoming table
 *                  (any hashbits and depth; its maxtimebits must be the device table's)
 *   id_offset      len(self.names) before this merge: every incoming entry moves up by
 *                  id_offset << maxtimebits (uint32), which must stay below 2^32
 *   np_state625    NumPy's legacy MT19937 state, np.random.get_state()[1] (624 words) then [2] (the
 *                  position); updated in place as the reference's np.random.permutation calls leave it
 *   noverflow      HOST, may be NULL: number of buckets that overflowed (and drew)
 *   stage_ms       HOST double [6] or NULL: incoming upload, classify + compaction, host replay,
 *                  pool-index uploads, apply kernels (CUDA events), wait after the last replay.
 *                  With stage_ms the upload and the classify step are synchronised to be timed.
 * For every incoming bucket with a non-zero count, in ascending order: pool = our first
 * min(count, depth) entries then its first min(count, its depth) shifted entries; a pool of at most
 * `depth` entries is written from slot 0 (later slots keep their values) and becomes the count; a
 * larger one gets table[b] = np.random.permutation(pool)[:depth] and counts[b] += its count (raw).
 * AFP_ERR_INDEX when a non-zero count of the incoming table lies outside the device table,
 * AFP_ERR_INVALID for a negative incoming count; both are found before anything changes.  The
 * device hashesperid is not touched and the pruning bound is 0 (no pruning) until
 * afp_table_set_hashesperid uploads the merged one. */
int afp_table_merge(afp_ctx* ctx, const uint32_t* table, const int32_t* counts, int32_t hashbits, int32_t depth,
                    int64_t id_offset, uint32_t* np_state625, int64_t* noverflow, double* stage_ms);
/* afp_table_merge with the incoming table in DEVICE memory (same arguments, same result, same
 * errors): table_dev uint32 [2^hashbits][depth] and counts_dev int32 [2^hashbits], e.g. a table
 * exported by afp_table_export on this or another GPU.  The rows are read in place; only the counts
 * are copied to the host, for the checks, which fail (AFP_ERR_INVALID / AFP_ERR_INDEX) before anything
 * changes.  stage_ms[0] is that copy.  The buffers are no longer read when the call returns. */
int afp_table_merge_device(afp_ctx* ctx, const uint32_t* table_dev, const int32_t* counts_dev, int32_t hashbits,
                           int32_t depth, int64_t id_offset, uint32_t* np_state625, int64_t* noverflow,
                           double* stage_ms);
/* Device-to-device copy of the device table into caller-owned DEVICE buffers: table_dev uint32
 * [2^hashbits][depth], counts_dev int32 [2^hashbits] (the geometry of the last upload / create).
 * Synchronises before it returns, so the buffers may go straight to a transfer on another stream. */
int afp_table_export(afp_ctx* ctx, uint32_t* table_dev, int32_t* counts_dev);
/* np.random.permutation of n pools (hash_table.py:291-323, the draws of HashTable.merge), replayed
 * on index arrays: out (HOST int32 [n][keep]) receives the first `keep` entries of the permutation of
 * 0..pool_sizes[i]-1 that RandomState.permutation would return for a pool of that size, the pools in
 * order from the state state625 (as in afp_table_merge), which is advanced in place.  Host
 * arithmetic only.  AFP_ERR_INVALID, state unchanged, for keep < 1 or a pool size below keep. */
int afp_np_permutation_replay(uint32_t* state625, const int32_t* pool_sizes, int64_t n, int32_t keep, int32_t* out);
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
 *       5 candidate depth > 1024, 7 more than 2048 members at or above the weight bin of the
 *       K-th member, 8 internal consistency check), 6 = the long-query path finished it
 *       (columns 1-7 are 0 then), -1 = the fast kernel did not run;
 *   [1] multi-record ids, [2] their hits, [3] single-record ids admitted by pass 3,
 *   [4] candidate depth, [5] ids above threshcount, [6] largest bucket multiplicity, [7] distinct
 *       ids (shard mode only). */
int afp_fetch_match_status(afp_ctx* ctx, int32_t* status);
/* After afp_match_batch with publish_candidates = 1: `cand` float64
 * [nqueries][search_depth][3] = (id, raw count, weighted count) in (weight desc, id desc)
 * order, `counts` int32 [nqueries][2] = (entries used, #ids with raw > threshcount). */
int afp_fetch_match_candidates(afp_ctx* ctx, double* cand, int32_t* counts, int on_host);
/* Matcher.match_hashes with exact_count and/or find_time_range (audfprint_match.py:149-244) for a
 * batch, finished on the device without materialising the hits.  Same query and matcher arguments
 * as afp_match_batch; the queries are ranked in publish mode (publish_candidates is implied), then
 *   exact_count      rows (id, distinct (qtime, hash) keys within +-window of the mode, mode, raw,
 *                    rank, tmin, tmax) for every histogram mode >= threshcount of every candidate of
 *                    rank < min(n_above, search_depth) whose count >= threshcount - no
 *                    max_alignments_per_id cap and no row capacity;
 *   find_time_range  columns 5-6 = the quantile-trimmed query times of each row's support
 *                    (t[int(n*q)], t[int(n*(1-q)) - 1], Python index semantics); without exact_count
 *                    the rows are afp_match_batch's (row_capacity applies as there).
 * timebits_breaks  HOST int64 [32]: entry k-1 = the smallest qmax for which the host's
 *                  ceil(log(qmax)/log(2)) >= k; a query's packed keys use max(1, #entries <= its
 *                  largest qtime) bits, as the reference does (power-of-two shortfall included).
 * Rows in (query, candidate rank, mode) order via afp_fetch_match_rows, the ranked candidates via
 * afp_fetch_match_candidates.  AFP_ERR_INDEX when a quantile index leaves its support. */
int afp_match_options_batch(afp_ctx* ctx, const int32_t* q_rows, int q_on_host, int32_t nqueries,
                            const int64_t* q_offsets, const afp_matcher_params* p, int32_t exact_count,
                            int32_t find_time_range, double time_quantile, const int64_t* timebits_breaks,
                            int64_t* total_rows);

/* ---- table sharded by track-id range (SURVEY.md 8e; BASELINE configs[4]) -----------------
 * The reference has no such mode; the nearest thing is one table per worker process merged
 * afterwards (audfprint.py:199-235, hash_table.py:291-323).  Every rank uploads the table,
 * keeps its id range (afp_table_restrict_ids), runs afp_match_batch with publish_candidates = 1
 * on ALL queries, packs one fixed-size record per query into a caller-owned DEVICE buffer, the
 * caller all-gathers the buffers (NCCL), and afp_shard_merge rebuilds on the device the rows a
 * single table would give (same rows, same ranks); fetch them with afp_fetch_match_rows.
 * Record (little endian): int32 {n_above, ncand, nrows, status}; f64 weight[sd]; uint32 id[sd];
 * uint32 raw[sd]; int32 rows[row_cap][7].  row_cap must be even.
 *
 * exact_count / find_time_range on a sharded table (audfprint_match.py:149-244): the reference
 * finishes each candidate from that candidate's hits alone, and a track id lives in one shard, so
 * a shard can finish its own ids - given three things that are not local:
 *   - depth: the whole table finishes ranks < D = min(sum n_above, search_depth); a shard's id can
 *     be inside the global top-D at or past its shard's n_above, so a shard finishes every
 *     candidate it publishes (rank < min(entries, search_depth)) and the merge drops ranks >= D;
 *   - key width: the packed (qtime, hash) keys take ceil(log(qmax)/log(2)) bits of the query's
 *     largest qtime over ALL its hits (:157-167), the maximum over the shards of the shard maxima;
 *   - errors: a quantile index outside its support (IndexError, :184-188) counts only at a global
 *     rank < D, and a rank must not fail between the collectives; the shard records it instead.
 * Hence two calls around one all-reduce (MAX) of one int32 per query:
 *   afp_match_options_shard_rank    the ranking of afp_match_options_batch (same arguments), then
 *                                   writes each query's largest qtime over the rows whose bucket is
 *                                   non-empty on this shard into the CALLER's device int32
 *                                   qmax_dev[nqueries] (the caller all-reduces it in place; no other
 *                                   call on the context in between, and device query rows must
 *                                   stay valid until the finish);
 *   afp_match_options_shard_finish  the finish with that depth rule and the reduced qmax_dev;
 *                                   fails only for reasons that are not data-dependent.
 * afp_shard_pack then packs the finished rows (nrows = the rows the shard produced, which may
 * exceed row_cap) and the status word: bit 0 = more rows than row_cap, bits 1-30 = 1 + the
 * smallest local rank whose quantile read failed.  afp_shard_merge returns AFP_ERR_INDEX when such
 * a candidate's global rank is < D, else AFP_ERR_INVALID ("row capacity: ...") when any record
 * overflowed - the same outcome on every rank, as every rank merges the same bytes.  After a
 * plain afp_match_batch the status word is 0 and an overflow fails afp_shard_pack itself. */
int afp_match_options_shard_rank(afp_ctx* ctx, const int32_t* q_rows, int q_on_host, int32_t nqueries,
                                 const int64_t* q_offsets, const afp_matcher_params* p, int32_t exact_count,
                                 int32_t find_time_range, double time_quantile,
                                 const int64_t* timebits_breaks, int32_t* qmax_dev, int64_t* ranked_rows);
int afp_match_options_shard_finish(afp_ctx* ctx, const int32_t* qmax_dev, int64_t* total_rows);
int64_t afp_shard_record_bytes(int32_t search_depth, int32_t row_cap);
int afp_shard_pack(afp_ctx* ctx, int32_t row_cap, void* records_dev /* [nqueries][record bytes] */);
int afp_shard_merge(afp_ctx* ctx, const void* gathered_dev /* [nshards][nqueries][record bytes] */,
                    int32_t nshards, int32_t nqueries, int32_t search_depth, int32_t row_cap,
                    int64_t* total_rows);

#ifdef __cplusplus
}
#endif
#endif /* AFP_H_ */
