// C ABI of libafp.so (see include/afp.h): context, analyzer configuration and
// the fingerprint batch driver.  Table / match entry points are in afp_match.cu.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <new>

#include "afp_internal.cuh"

int afp_write_hashes(afp_ctx* c);

extern "C" {

int afp_abi_version(void) { return AFP_ABI_VERSION; }

int afp_create(afp_ctx** out, int device) {
  if (!out) return AFP_ERR_INVALID;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return AFP_ERR_CUDA;   // no CPU fallback
  if (device < 0 || device >= ndev) return AFP_ERR_INVALID;
  if (cudaSetDevice(device) != cudaSuccess) return AFP_ERR_CUDA;
  afp_ctx* c = new (std::nothrow) afp_ctx();
  if (!c) return AFP_ERR_NOMEM;
  c->device = device;
  if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete c;
    return AFP_ERR_CUDA;
  }
  c->own_stream = true;
  cudaDeviceGetAttribute(&c->num_sms, cudaDevAttrMultiProcessorCount, device);
  // double2 tables: tw256[p][r] = W256^(r p); W512^k (k < 256); log table (c_i, -0.5 log c_i) x 8 copies
  std::vector<double> tw(2 * (256 + 256 + 64 * 8));
  const long double pi = 3.14159265358979323846264338327950288L;
  for (int p = 0; p < 16; ++p)
    for (int r = 0; r < 16; ++r) {
      const int e = (r * p) & 255;
      tw[2 * (p * 16 + r)] = (double)cosl(2.0L * pi * e / 256.0L);
      tw[2 * (p * 16 + r) + 1] = (double)(-sinl(2.0L * pi * e / 256.0L));
    }
  for (int k = 0; k < 256; ++k) {
    tw[512 + 2 * k] = (double)cosl(2.0L * pi * k / 512.0L);
    tw[512 + 2 * k + 1] = (double)(-sinl(2.0L * pi * k / 512.0L));
  }
  for (int i = 0; i < 64; ++i) {   // 8 interleaved copies: entry i of copy j at [i * 8 + j]
    const double ci = (double)(1.0L / (1.0L + (i + 0.5L) / 64.0L));
    for (int j = 0; j < 8; ++j) {
      tw[1024 + 2 * (i * 8 + j)] = ci;
      tw[1024 + 2 * (i * 8 + j) + 1] = (double)(-0.5L * logl((long double)ci));
    }
  }
  std::vector<float> twf(2 * 512);
  for (size_t i = 0; i < twf.size(); ++i) twf[i] = (float)tw[i];
  if (c->d_twid.reserve(tw.size() * sizeof(double)) != cudaSuccess ||
      cudaMemcpy(c->d_twid.p, tw.data(), tw.size() * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess ||
      c->d_twid_f.reserve(twf.size() * sizeof(float)) != cudaSuccess ||
      cudaMemcpy(c->d_twid_f.p, twf.data(), twf.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
    afp_destroy(c);
    return AFP_ERR_CUDA;
  }
  *out = c;
  return AFP_OK;
}

void afp_destroy(afp_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  for (int i = 0; i <= AFP_NSTAGES; ++i)
    if (c->ev[i]) cudaEventDestroy(c->ev[i]);
  DevBuf* bufs[] = {&c->d_window, &c->d_window_f, &c->d_twid_f, &c->d_gauss, &c->d_twid, &c->d_pcm_stage, &c->d_items, &c->d_tile_item, &c->d_file_col_base,
                    &c->d_logs, &c->d_nyq, &c->d_tile_stats, &c->d_item_stats, &c->d_fwd_val, &c->d_fwd_bin,
                    &c->d_fwd_cnt, &c->d_pk_bin, &c->d_pk_cnt, &c->d_item_scols, &c->d_item_npeaks, &c->d_lm,
                    &c->d_col_cnt, &c->d_file_tot, &c->d_file_off, &c->d_hashes, &c->d_pk_off, &c->d_pk_rows,
                    &c->d_tmp, &c->tab.table, &c->tab.counts, &c->tab.hashesperid, &c->d_q, &c->d_qoff,
                    &c->d_hit_off, &c->d_hits, &c->d_st_off, &c->d_st_ids, &c->d_st_eval, &c->d_st_seq, &c->d_st_ovf,
                    &c->d_st_cnt, &c->d_st_seg, &c->d_st_heavy, &c->d_st_part, &c->d_st_scan, &c->d_st_obkt,
                    &c->d_st_opos, &c->d_st_oval, &c->d_st_slot, &c->d_st_last, &c->d_mfast, &c->d_mqlist, &c->d_mscratch, &c->d_mrows, &c->d_mrow_cnt,
                    &c->d_mrow_off, &c->d_mrows_packed, &c->d_mcand, &c->d_mcand_cnt,
                    &c->d_ed_ids, &c->d_ed_bits, &c->d_ed_slot, &c->d_ed_cnt, &c->d_ed_off, &c->d_ed_key,
                    &c->d_ed_key2, &c->d_ed_val, &c->d_ed_val2, &c->d_ed_cub, &c->d_ed_uoff, &c->d_ed_req,
                    &c->d_ed_rows, &c->d_lg_key, &c->d_lg_cub, &c->d_lg_id, &c->d_lg_w, &c->d_lg_cand,
                    &c->d_lg_dts, &c->d_lg_hist};
  for (DevBuf* b : bufs) b->release();
  if (c->copy_stream) {
    cudaStreamDestroy(c->copy_stream);
    for (auto& e : c->ev_chunk) if (e) cudaEventDestroy(e);
    if (c->ev_batch_done) cudaEventDestroy(c->ev_batch_done);
    for (int i = 0; i < 4; ++i) {
      if (c->chunk_stream[i]) cudaStreamDestroy(c->chunk_stream[i]);
      if (c->ev_chunk_stream[i]) cudaEventDestroy(c->ev_chunk_stream[i]);
    }
  }
  if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
  delete c;
}

const char* afp_last_error(afp_ctx* c) { return c ? c->err.c_str() : "null context"; }

int afp_set_stream(afp_ctx* c, void* s) {
  if (!c) return AFP_ERR_INVALID;
  AFP_CUDA(c, cudaSetDevice(c->device));
  if (c->own_stream && c->stream) {
    cudaStreamSynchronize(c->stream);
    cudaStreamDestroy(c->stream);
  }
  if (s) {
    c->stream = static_cast<cudaStream_t>(s);
    c->own_stream = false;
  } else {
    AFP_CUDA(c, cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    c->own_stream = true;
  }
  return AFP_OK;
}

int afp_sync(afp_ctx* c) {
  if (!c) return AFP_ERR_INVALID;
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  return AFP_OK;
}

int64_t afp_launch_count(afp_ctx* c) { return c ? c->launches : -1; }

int afp_set_profiling(afp_ctx* c, int enable) {
  if (!c) return AFP_ERR_INVALID;
  AFP_CUDA(c, cudaSetDevice(c->device));
  if (enable && !c->ev[0])
    for (int i = 0; i <= AFP_NSTAGES; ++i) AFP_CUDA(c, cudaEventCreate(&c->ev[i]));
  c->profiling = enable != 0;
  c->ev_valid = false;
  return AFP_OK;
}

int afp_get_stage_ms(afp_ctx* c, float* ms) {
  if (!c || !ms) return AFP_ERR_INVALID;
  if (!c->ev_valid) AFP_FAIL(c, AFP_ERR_STATE, "no profiled batch");
  AFP_CUDA(c, cudaEventSynchronize(c->ev[AFP_NSTAGES]));
  for (int i = 0; i < AFP_NSTAGES; ++i) AFP_CUDA(c, cudaEventElapsedTime(&ms[i], c->ev[i], c->ev[i + 1]));
  return AFP_OK;
}

int afp_set_analyzer(afp_ctx* c, const afp_analyzer_params* p, const double* window, const double* gauss,
                     double f_sd) {
  if (!c || !p) return AFP_ERR_INVALID;
  AFP_CUDA(c, cudaSetDevice(c->device));
  if (p->maxpksperframe < 1 || p->maxpksperframe > AFP_MAX_PKS)
    AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "maxpksperframe must be in [1, 16]");
  if (p->maxpairsperpeak < 1 || p->shifts < 1 ||
      (int64_t)p->shifts * p->maxpksperframe * p->maxpairsperpeak > AFP_MAX_MERGE)
    AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "shifts*maxpksperframe*maxpairsperpeak must be in [1, 256]");
  if (p->mindt < 0 || p->targetdt <= p->mindt || p->targetdt > 64 || p->targetdf < 1 || p->targetdf > 32)
    AFP_FAIL(c, AFP_ERR_INVALID, "pairing window outside the 6-bit hash fields");
  if (!(p->a_dec > 0.0) || !(f_sd > 0.0 || gauss)) AFP_FAIL(c, AFP_ERR_INVALID, "bad a_dec / f_sd");
  std::vector<double> w(2 * AFP_N_FFT), g(AFP_GAUSS_N);
  const double pi = 3.14159265358979323846;
  for (int k = 0; k < AFP_N_FFT; ++k) {   // np.hanning(514)[1:-1]
    w[k] = window ? window[k] : 0.5 - 0.5 * cos(2.0 * pi * (k + 1) / (AFP_N_FFT + 1));
    w[AFP_N_FFT + k] = w[k] * (1.0 / 32768.0);   // exact: (x/32768)*w == x*(w/32768)
  }
  for (int j = 0; j < AFP_GAUSS_N; ++j) {
    const double u = (double)(j - AFP_NBINS) / f_sd;
    g[j] = gauss ? gauss[j] : exp(-0.5 * (u * u));
  }
  AFP_CUDA(c, c->d_window.reserve(w.size() * sizeof(double)));
  AFP_CUDA(c, c->d_gauss.reserve(g.size() * sizeof(double)));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  AFP_CUDA(c, cudaMemcpy(c->d_window.p, w.data(), w.size() * sizeof(double), cudaMemcpyHostToDevice));
  std::vector<float> wf(w.size());
  for (size_t i = 0; i < w.size(); ++i) wf[i] = (float)w[i];
  AFP_CUDA(c, c->d_window_f.reserve(wf.size() * sizeof(float)));
  AFP_CUDA(c, cudaMemcpy(c->d_window_f.p, wf.data(), wf.size() * sizeof(float), cudaMemcpyHostToDevice));
  AFP_CUDA(c, cudaMemcpy(c->d_gauss.p, g.data(), g.size() * sizeof(double), cudaMemcpyHostToDevice));
  c->ap = *p;
  c->analyzer_set = true;
  c->batch_valid = false;
  return AFP_OK;
}

}  // extern "C"

// Size the workspace for the batch described by h_items / h_file_col_base and the totals
// (afp_fingerprint_batch, afp_sgram, afp_fingerprint_from_logs), and upload its item table.
static int reserve_batch(afp_ctx* c) {
  const int32_t nfiles = c->nfiles;
  const int64_t frames = c->total_frames, tiles = c->total_tiles, cols = c->total_cols;
  const size_t P = (size_t)c->ap.maxpksperframe, F = (size_t)c->ap.maxpairsperpeak;
  const size_t fr = (size_t)frames + 1;
  AFP_CUDA(c, c->d_items.reserve(sizeof(ItemDesc) * (size_t)(c->nitems + 1)));
  AFP_CUDA(c, c->d_file_col_base.reserve(sizeof(int64_t) * (size_t)(nfiles + 1)));
  AFP_CUDA(c, c->d_tile_item.reserve(sizeof(int32_t) * (size_t)(tiles + 1)));
  AFP_CUDA(c, c->d_logs.reserve(sizeof(double) * AFP_NBINS * fr));
  AFP_CUDA(c, c->d_nyq.reserve(sizeof(double) * fr));
  AFP_CUDA(c, c->d_tile_stats.reserve(sizeof(double) * 3 * (size_t)(tiles + 1)));
  AFP_CUDA(c, c->d_item_stats.reserve(sizeof(ItemStats) * (size_t)(c->nitems + 1)));
  AFP_CUDA(c, c->d_fwd_val.reserve(sizeof(double) * P * fr));
  AFP_CUDA(c, c->d_fwd_bin.reserve(P * fr));
  AFP_CUDA(c, c->d_fwd_cnt.reserve(fr));
  AFP_CUDA(c, c->d_pk_bin.reserve(P * fr));
  AFP_CUDA(c, c->d_pk_cnt.reserve(fr));
  AFP_CUDA(c, c->d_item_scols.reserve(sizeof(int32_t) * (size_t)(c->nitems + 1)));
  AFP_CUDA(c, c->d_item_npeaks.reserve(sizeof(int32_t) * (size_t)(c->nitems + 1)));
  AFP_CUDA(c, c->d_lm.reserve(sizeof(uint32_t) * P * F * fr));
  AFP_CUDA(c, c->d_col_cnt.reserve(sizeof(int32_t) * (size_t)(cols + 1)));
  AFP_CUDA(c, c->d_file_tot.reserve(sizeof(int32_t) * (size_t)(nfiles + 1)));
  AFP_CUDA(c, c->d_file_off.reserve(sizeof(int64_t) * (size_t)(nfiles + 1)));
  // upper bound on the output: every hash slot distinct
  AFP_CUDA(c, c->d_hashes.reserve(sizeof(int32_t) * 2 * (P * F * fr + 1)));
  if (c->nitems > 0)
    AFP_CUDA(c, cudaMemcpyAsync(c->d_items.p, c->h_items.data(), sizeof(ItemDesc) * (size_t)c->nitems,
                                cudaMemcpyHostToDevice, c->stream));
  AFP_CUDA(c, cudaMemcpyAsync(c->d_file_col_base.p, c->h_file_col_base.data(),
                              sizeof(int64_t) * (size_t)(nfiles + 1), cudaMemcpyHostToDevice, c->stream));
  return AFP_OK;
}

// Build the item table of a batch, size the workspace, stage the PCM.
static int prepare_batch(afp_ctx* c, const void* pcm, int dtype, int on_host, int32_t nfiles,
                         const int64_t* off, const int64_t* lens, int shifts, const void** pcm_dev,
                         bool chunked = false) {
  if (dtype != AFP_PCM_I16 && dtype != AFP_PCM_F32) AFP_FAIL(c, AFP_ERR_INVALID, "unknown pcm dtype");
  if (nfiles < 0 || (nfiles > 0 && (!off || !pcm))) AFP_FAIL(c, AFP_ERR_INVALID, "null pcm / offsets");
  for (int f = 0; f < nfiles; ++f) {
    if (off[f + 1] < off[f]) AFP_FAIL(c, AFP_ERR_INVALID, "sample_offsets must be non-decreasing");
    if (lens && (lens[f] < 0 || lens[f] > off[f + 1] - off[f]))
      AFP_FAIL(c, AFP_ERR_INVALID, "sample_lengths[i] must be in [0, off[i+1]-off[i]]");
  }
  c->batch_valid = false;
  c->nfiles = nfiles;
  c->nitems = nfiles * shifts;
  c->pcm_dtype = dtype;
  c->h_items.resize((size_t)c->nitems);
  c->h_file_col_base.resize((size_t)nfiles + 1);
  int64_t frames = 0, tiles = 0, cols = 0;
  for (int f = 0; f < nfiles; ++f) {
    const int64_t len = lens ? lens[f] : off[f + 1] - off[f];
    c->h_file_col_base[f] = cols;
    for (int s = 0; s < shifts; ++s) {
      // int(shift / shifts * n_hop), audfprint_analyze.py:375
      const int64_t so = (int64_t)((double)s / (double)shifts * (double)AFP_N_HOP);
      ItemDesc& it = c->h_items[(size_t)f * shifts + s];
      it.sample_start = off[f] + so;
      it.nsamples = len - so;
      it.nframes = it.nsamples >= 1 ? (int32_t)(1 + it.nsamples / AFP_N_HOP) : 0;   // stft.py:33,88
      it.frame_base = frames;
      if (tiles > 0x7fffffff - 4096) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "batch too large (tile index)");
      it.tile_base = (int32_t)tiles;
      frames += it.nframes;
      tiles += (it.nframes + AFP_FRAMES_PER_TILE - 1) / AFP_FRAMES_PER_TILE;
      if (s == 0) cols += it.nframes;
    }
  }
  c->h_file_col_base[nfiles] = cols;
  c->total_frames = frames;
  c->total_tiles = tiles;
  c->total_cols = cols;
  int rc = reserve_batch(c);
  if (rc) return rc;
  *pcm_dev = pcm;
  if (on_host && nfiles > 0) {
    const size_t esz = dtype == AFP_PCM_I16 ? 2 : 4;
    const size_t bytes = (size_t)(off[nfiles] - off[0]) * esz;
    AFP_CUDA(c, c->d_pcm_stage.reserve(bytes + 16));
    // staged copy starts at sample off[0]: rebase the pointer so that item offsets still apply
    *pcm_dev = (const char*)c->d_pcm_stage.p - (size_t)off[0] * esz;
    if (!chunked)
      AFP_CUDA(c, cudaMemcpyAsync(c->d_pcm_stage.p, (const char*)pcm + (size_t)off[0] * esz, bytes,
                                  cudaMemcpyHostToDevice, c->stream));
  }
  return AFP_OK;
}

// Host-resident PCM: copy the batch in file chunks on a second stream and start
// the kernels of a chunk as soon as its samples have landed, so that the PCIe
// transfer (the end-to-end bound: 22 KB per audio-second) overlaps the compute.
static int run_chunked(afp_ctx* c, const void* pcm, int dtype, int32_t nfiles, const int64_t* off,
                       const void* dpcm) {
  const size_t esz = dtype == AFP_PCM_I16 ? 2 : 4;
  const int S = c->ap.shifts;
  if (!c->copy_stream) {
    AFP_CUDA(c, cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    for (auto& e : c->ev_chunk) AFP_CUDA(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    AFP_CUDA(c, cudaEventCreateWithFlags(&c->ev_batch_done, cudaEventDisableTiming));
    for (int i = 0; i < 4; ++i) {
      AFP_CUDA(c, cudaStreamCreateWithFlags(&c->chunk_stream[i], cudaStreamNonBlocking));
      AFP_CUDA(c, cudaEventCreateWithFlags(&c->ev_chunk_stream[i], cudaEventDisableTiming));
    }
  }
  const size_t total = (size_t)(off[nfiles] - off[0]) * esz;
  // K2's duration is set by the file length, not by the number of files, so chunks are
  // few and their kernel chains run on 4 streams so that the K2s of different chunks overlap
  int nch = (int)std::min<size_t>(8, std::max<size_t>(1, total / ((size_t)40 << 20)));
  nch = std::min(nch, nfiles);
  // the staging buffer may still be read by the previous batch's kernels
  AFP_CUDA(c, cudaEventRecord(c->ev_batch_done, c->stream));
  AFP_CUDA(c, cudaStreamWaitEvent(c->copy_stream, c->ev_batch_done, 0));
  for (int i = 0; i < 4; ++i) AFP_CUDA(c, cudaStreamWaitEvent(c->chunk_stream[i], c->ev_batch_done, 0));
  std::vector<int> fb(nch + 1, 0);
  int f = 0;
  for (int k = 0; k < nch; ++k) {
    fb[k] = f;
    const size_t target = (size_t)off[0] * esz + total * (size_t)(k + 1) / (size_t)nch;
    while (f < nfiles && ((size_t)off[f + 1] * esz <= target || f == fb[k])) ++f;
    if (k == nch - 1) f = nfiles;
    const size_t b0 = (size_t)off[fb[k]] * esz, b1 = (size_t)off[f] * esz;
    if (b1 > b0)
      AFP_CUDA(c, cudaMemcpyAsync((char*)c->d_pcm_stage.p + (b0 - (size_t)off[0] * esz), (const char*)pcm + b0,
                                  b1 - b0, cudaMemcpyHostToDevice, c->copy_stream));
    AFP_CUDA(c, cudaEventRecord(c->ev_chunk[k], c->copy_stream));
  }
  fb[nch] = nfiles;
  int rc;
  if ((rc = afp_launch_tile_table(c))) return rc;
  AFP_CUDA(c, cudaEventRecord(c->ev_batch_done, c->stream));   // item + tile tables are in place
  for (int i = 0; i < 4; ++i) AFP_CUDA(c, cudaStreamWaitEvent(c->chunk_stream[i], c->ev_batch_done, 0));
  cudaStream_t user = c->stream;
  for (int k = 0; k < nch; ++k) {
    const int f0 = fb[k], f1 = fb[k + 1];
    if (f1 <= f0) continue;
    c->stream = c->chunk_stream[k & 3];          // launchers issue on c->stream
    cudaError_t e = cudaStreamWaitEvent(c->stream, c->ev_chunk[k], 0);
    const int i0 = f0 * S, i1 = f1 * S;
    const int64_t t0 = c->h_items[i0].tile_base;
    const int64_t t1 = (i1 < c->nitems) ? c->h_items[i1].tile_base : c->total_tiles;
    rc = (e == cudaSuccess) ? AFP_OK : AFP_ERR_CUDA;
    if (!rc) rc = afp_launch_stft(c, dpcm, dtype, nullptr, t0, t1 - t0);
    if (!rc) rc = afp_launch_stats(c, i0, i1 - i0);
    if (!rc) rc = afp_launch_peaks(c, i0, i1 - i0);
    if (!rc) rc = afp_launch_landmarks(c, i0, i1 - i0);
    c->stream = user;
    if (rc) return rc;
  }
  for (int i = 0; i < 4; ++i) {
    AFP_CUDA(c, cudaEventRecord(c->ev_chunk_stream[i], c->chunk_stream[i]));
    AFP_CUDA(c, cudaStreamWaitEvent(c->stream, c->ev_chunk_stream[i], 0));
  }
  if ((rc = afp_launch_hashes(c))) return rc;
  return afp_write_hashes(c);
}

extern "C" {

int afp_fingerprint_batch(afp_ctx* c, const void* pcm, int pcm_dtype, int pcm_on_host, int32_t nfiles,
                          const int64_t* sample_offsets, const int64_t* sample_lengths, int64_t* total_hashes) {
  if (!c) return AFP_ERR_INVALID;
  if (!c->analyzer_set) AFP_FAIL(c, AFP_ERR_STATE, "afp_set_analyzer has not been called");
  AFP_CUDA(c, cudaSetDevice(c->device));
  const void* dpcm = nullptr;
#define AFP_MARK(i) do { if (c->profiling) AFP_CUDA(c, cudaEventRecord(c->ev[i], c->stream)); } while (0)
  c->ev_valid = false;
  const bool chunked = pcm_on_host && nfiles > 1 && !c->profiling &&
                       (sample_offsets[nfiles] - sample_offsets[0]) * (pcm_dtype == AFP_PCM_I16 ? 2 : 4) >= (64 << 20);
  AFP_MARK(0);
  int rc = prepare_batch(c, pcm, pcm_dtype, pcm_on_host, nfiles, sample_offsets, sample_lengths, c->ap.shifts, &dpcm,
                         chunked);
  if (rc) return rc;
  c->total_hashes = -1;
  if (chunked) {
    if ((rc = run_chunked(c, pcm, pcm_dtype, nfiles, sample_offsets, dpcm))) return rc;
  } else {
    AFP_MARK(1);
    if ((rc = afp_launch_tile_table(c))) return rc;
    if ((rc = afp_launch_stft(c, dpcm, pcm_dtype, nullptr, 0, c->total_tiles))) return rc;
    AFP_MARK(2);
    if ((rc = afp_launch_stats(c, 0, c->nitems))) return rc;
    AFP_MARK(3);
    if ((rc = afp_launch_peaks(c, 0, c->nitems))) return rc;
    AFP_MARK(4);
    if ((rc = afp_launch_landmarks(c, 0, c->nitems))) return rc;
    if ((rc = afp_launch_hashes(c))) return rc;
    if ((rc = afp_write_hashes(c))) return rc;
    AFP_MARK(5);
    c->ev_valid = c->profiling;
  }
#undef AFP_MARK
  c->batch_valid = true;
  if (total_hashes) {
    AFP_CUDA(c, cudaMemcpyAsync(&c->total_hashes, c->d_file_off.as<int64_t>() + nfiles, sizeof(int64_t),
                                cudaMemcpyDeviceToHost, c->stream));
    AFP_CUDA(c, cudaStreamSynchronize(c->stream));
    *total_hashes = c->total_hashes;
  }
  return AFP_OK;
}

int afp_fingerprint_from_logs(afp_ctx* c, const void* logs, int logs_on_host, int32_t nfiles,
                              const int32_t* item_frames, const double* item_stats, int64_t* total_hashes) {
  if (!c) return AFP_ERR_INVALID;
  if (!c->analyzer_set) AFP_FAIL(c, AFP_ERR_STATE, "afp_set_analyzer has not been called");
  if (nfiles < 0 || (nfiles > 0 && (!item_frames || !item_stats)))
    AFP_FAIL(c, AFP_ERR_INVALID, "null item frames / stats");
  const int S = c->ap.shifts;
  int64_t frames = 0;
  for (int f = 0; f < nfiles; ++f)
    for (int s = 0; s < S; ++s) {
      const int32_t n = item_frames[(size_t)f * S + s];
      if (n < 0) AFP_FAIL(c, AFP_ERR_INVALID, "item frame counts must be >= 0");
      if (n > item_frames[(size_t)f * S]) AFP_FAIL(c, AFP_ERR_INVALID, "a shift item is longer than shift 0");
      frames += n;
    }
  if (frames > 0 && !logs) AFP_FAIL(c, AFP_ERR_INVALID, "null logs");
  AFP_CUDA(c, cudaSetDevice(c->device));
  c->batch_valid = false;
  c->ev_valid = false;
  c->total_hashes = -1;
  c->nfiles = nfiles;
  c->nitems = nfiles * S;
  c->h_items.assign((size_t)c->nitems, ItemDesc{});
  c->h_file_col_base.resize((size_t)nfiles + 1);
  std::vector<ItemStats> st((size_t)c->nitems);
  int64_t base = 0, cols = 0;
  for (int i = 0; i < c->nitems; ++i) {
    ItemDesc& it = c->h_items[(size_t)i];
    it.nframes = item_frames[i];
    it.frame_base = base;
    base += it.nframes;
    if (i % S == 0) {
      c->h_file_col_base[(size_t)i / S] = cols;
      cols += it.nframes;
    }
    st[(size_t)i] = ItemStats{item_stats[3 * i], item_stats[3 * i + 1], item_stats[3 * i + 2] != 0.0 ? 1 : 0, 0};
  }
  c->h_file_col_base[(size_t)nfiles] = cols;
  c->total_frames = frames;
  c->total_tiles = 0;
  c->total_cols = cols;
  int rc = reserve_batch(c);
  if (rc) return rc;
  // K2 bulk-copies its columns out of d_logs, as it does after K1
  const size_t esz = c->ap.spectrogram_fp32 ? sizeof(float) : sizeof(double);
  if (frames > 0)
    AFP_CUDA(c, cudaMemcpyAsync(c->d_logs.p, logs, esz * AFP_NBINS * (size_t)frames,
                                logs_on_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, c->stream));
  if (c->nitems > 0)
    AFP_CUDA(c, cudaMemcpyAsync(c->d_item_stats.p, st.data(), sizeof(ItemStats) * st.size(), cudaMemcpyHostToDevice,
                                c->stream));
  if ((rc = afp_launch_peaks(c, 0, c->nitems))) return rc;
  if ((rc = afp_launch_landmarks(c, 0, c->nitems))) return rc;
  if ((rc = afp_launch_hashes(c))) return rc;
  if ((rc = afp_write_hashes(c))) return rc;
  c->batch_valid = true;
  c->total_hashes = 0;
  if (nfiles > 0)
    AFP_CUDA(c, cudaMemcpyAsync(&c->total_hashes, c->d_file_off.as<int64_t>() + nfiles, sizeof(int64_t),
                                cudaMemcpyDeviceToHost, c->stream));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));   // `st` and host logs must outlive their copies
  if (total_hashes) *total_hashes = c->total_hashes;
  return AFP_OK;
}

int afp_fetch_hashes(afp_ctx* c, int32_t* rows, int rows_on_host, int64_t* row_offsets) {
  if (!c) return AFP_ERR_INVALID;
  if (!c->batch_valid) AFP_FAIL(c, AFP_ERR_STATE, "no fingerprint batch to fetch");
  AFP_CUDA(c, cudaSetDevice(c->device));
  if (c->total_hashes < 0) {
    AFP_CUDA(c, cudaMemcpyAsync(&c->total_hashes, c->d_file_off.as<int64_t>() + c->nfiles, sizeof(int64_t),
                                cudaMemcpyDeviceToHost, c->stream));
    AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  }
  if (row_offsets)
    AFP_CUDA(c, cudaMemcpyAsync(row_offsets, c->d_file_off.p, sizeof(int64_t) * (size_t)(c->nfiles + 1),
                                cudaMemcpyDeviceToHost, c->stream));
  if (rows && c->total_hashes > 0)
    AFP_CUDA(c, cudaMemcpyAsync(rows, c->d_hashes.p, sizeof(int32_t) * 2 * (size_t)c->total_hashes,
                                rows_on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, c->stream));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  return AFP_OK;
}

int afp_fetch_peaks(afp_ctx* c, int32_t shift, int32_t* rows, int rows_on_host, int64_t* row_offsets) {
  if (!c) return AFP_ERR_INVALID;
  if (!c->batch_valid) AFP_FAIL(c, AFP_ERR_STATE, "no fingerprint batch to fetch");
  if (shift < 0 || shift >= c->ap.shifts) AFP_FAIL(c, AFP_ERR_INVALID, "shift out of range");
  AFP_CUDA(c, cudaSetDevice(c->device));
  int rc = afp_compact_peaks(c, shift);
  if (rc) return rc;
  std::vector<int64_t> off((size_t)c->nfiles + 1);
  AFP_CUDA(c, cudaMemcpyAsync(off.data(), c->d_pk_off.p, sizeof(int64_t) * off.size(), cudaMemcpyDeviceToHost,
                              c->stream));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  if (row_offsets) memcpy(row_offsets, off.data(), sizeof(int64_t) * off.size());
  if (rows && off[c->nfiles] > 0)
    AFP_CUDA(c, cudaMemcpyAsync(rows, c->d_pk_rows.p, sizeof(int32_t) * 2 * (size_t)off[c->nfiles],
                                rows_on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, c->stream));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  return AFP_OK;
}

int afp_landmarks_from_peaks(afp_ctx* c, const int32_t* peak_rows, int64_t npeaks, int on_host,
                             int64_t* nlandmarks) {
  if (!c || npeaks < 0 || (npeaks > 0 && !peak_rows)) return AFP_ERR_INVALID;
  if (!c->analyzer_set) AFP_FAIL(c, AFP_ERR_STATE, "afp_set_analyzer has not been called");
  AFP_CUDA(c, cudaSetDevice(c->device));
  return afp_landmarks_from_peaks_impl(c, peak_rows, npeaks, on_host, nlandmarks);
}

int afp_fetch_landmarks(afp_ctx* c, int32_t* rows, int rows_on_host) {
  if (!c) return AFP_ERR_INVALID;
  if (c->nlandmarks < 0) AFP_FAIL(c, AFP_ERR_STATE, "afp_landmarks_from_peaks has not been called");
  AFP_CUDA(c, cudaSetDevice(c->device));
  if (rows && c->nlandmarks > 0)
    AFP_CUDA(c, cudaMemcpyAsync(rows, c->d_hashes.p, sizeof(int32_t) * 4 * (size_t)c->nlandmarks,
                                rows_on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, c->stream));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  return AFP_OK;
}

int afp_spread_peaks(afp_ctx* c, const double* vector, int32_t n, const double* table, double width,
                     const double* base, double* out) {
  if (!c || n < 0 || (n > 0 && (!vector || !out))) return AFP_ERR_INVALID;
  if (n == 0) return AFP_OK;
  if (n > 50000) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "spread_peaks: vector longer than 50000");
  if (!table && !(width > 0.0)) AFP_FAIL(c, AFP_ERR_INVALID, "spread_peaks: width must be positive");
  AFP_CUDA(c, cudaSetDevice(c->device));
  return afp_spread_peaks_impl(c, vector, n, table, width, base, out);
}

static int single_signal(afp_ctx* c, const void* pcm, int dtype, int on_host, int64_t n, double* out,
                         int out_on_host, bool want_mag) {
  if (!c) return AFP_ERR_INVALID;
  if (!c->analyzer_set) AFP_FAIL(c, AFP_ERR_STATE, "afp_set_analyzer has not been called");
  if (n < 1 || !out) AFP_FAIL(c, AFP_ERR_INVALID, "empty signal / null output");
  AFP_CUDA(c, cudaSetDevice(c->device));
  const int64_t off[2] = {0, n};
  const void* dpcm = nullptr;
  int rc = prepare_batch(c, pcm, dtype, on_host, 1, off, nullptr, 1, &dpcm);
  if (rc) return rc;
  const size_t T = (size_t)c->total_frames;
  const size_t width = want_mag ? 257 : AFP_NBINS;
  double* dout = out;
  if (out_on_host) {
    AFP_CUDA(c, c->d_tmp.reserve(sizeof(double) * width * T));
    dout = c->d_tmp.as<double>();
  }
  if ((rc = afp_launch_tile_table(c))) return rc;
  if ((rc = afp_launch_stft(c, dpcm, dtype, want_mag ? dout : nullptr, 0, c->total_tiles))) return rc;
  if (!want_mag) {
    if ((rc = afp_launch_stats(c, 0, c->nitems))) return rc;
    if ((rc = afp_launch_sgram(c, dout))) return rc;
  }
  if (out_on_host)
    AFP_CUDA(c, cudaMemcpyAsync(out, dout, sizeof(double) * width * T, cudaMemcpyDeviceToHost, c->stream));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  return AFP_OK;
}

int afp_stft_mag(afp_ctx* c, const void* pcm, int pcm_dtype, int pcm_on_host, int64_t n, double* mag,
                 int mag_on_host) {
  return single_signal(c, pcm, pcm_dtype, pcm_on_host, n, mag, mag_on_host, true);
}

int afp_sgram(afp_ctx* c, const void* pcm, int pcm_dtype, int pcm_on_host, int64_t n, double* sgram,
              int sgram_on_host) {
  return single_signal(c, pcm, pcm_dtype, pcm_on_host, n, sgram, sgram_on_host, false);
}

}  // extern "C"
