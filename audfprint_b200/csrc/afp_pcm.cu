// PCM front-end on the device (SURVEY.md §8f-2): interleaved int16 multi-channel PCM at any rate
// -> mono float32 at the analyzer's rate, i.e. what the reference has `ffmpeg -ac 1 -ar 11025`
// do before Analyzer ever sees a sample (audio_read.py:56-145, ffmpeg arguments :196-203) and what
// its reader then scales to [-1, 1) (audio_read.py:139-145).
//
//   mono[j] = mean over channels of pcm[j][c] / 32768                      (float32, as the reader yields)
//   out[n]  = sum_j taps[n*down + half - j*up] * mono[j]                   (polyphase FIR, zero phase)
// with the `up`-scaled Kaiser-windowed low-pass `taps` (2*half + 1 coefficients) computed by the
// host in float64 exactly as scipy.signal.resample_poly designs it; len(out) = ceil(n*up/down).
// The channel sum is exact in float32 (ch <= 512), so mono[j] is rounded once.  The FIR sums in
// float64, whose error (about m 2^-53 sum|t x| for m terms) is far below half a float32 ulp, so
// out[n] is the correctly rounded float32 of the exact sum except in a tie zone where that sum lies
// within the error bound of a rounding boundary.  tests/test_gpu_pcm_exact.py holds every output to
// that bar against the extended-precision statement of tests/exact_resample.py, which
// scipy.signal.resample_poly cross-checks on the CPU.  ffmpeg's resampler, which the reference uses,
// is not reproduced (§8f-2); parity statements against the reference are made on 11025 Hz PCM.
//
// afp_pcm_frontend_batch_bytes runs the same per-output function over a list of files in one launch,
// over packed payload bytes with a sample format per file: a 24-bit, 32-bit or float sample enters as
// the int16 `ffmpeg -ac 1` gives it at the file's own rate, at the sample load, so every format runs in
// the same launch.  The layout, checks, upload and launch it shares with the ffmpeg front-end
// (afp_pcm_formats.cuh); here are only the taps lookup and frontend_sample, and every distinct (up, down)
// design is uploaded once.  tests/test_gpu_pcm_batch.py holds it bit-equal to afp_pcm_frontend per file.
// The package calls only this byte form; afp_pcm_frontend_batch (int16) forwards to it, and
// afp_pcm_frontend keeps its single-file kernel for ABI callers and as the tests' per-file reference.
#include "afp_internal.cuh"
#include "afp_pcm_formats.cuh"

namespace {

__device__ __forceinline__ float mono_at(const uint8_t* pcm, int fmt, int64_t j, int ch) {
  float s = 0.0f;
  for (int c = 0; c < ch; ++c) s += (float)pcm_s16(pcm, fmt, j * ch + c) * (1.0f / 32768.0f);
  return ch == 1 ? s : s / (float)ch;
}

// Output n of one file: the down-mix alone (up = down = 1) or the polyphase FIR over it.  The single-file
// and the batched kernel both call this, so a file gives the same bits through either entry point.
__device__ __forceinline__ float frontend_sample(const uint8_t* pcm, int fmt, int64_t nframes, int ch, int up,
                                                 int down, const double* taps, int half, int64_t n) {
  if (up == 1 && down == 1) return mono_at(pcm, fmt, n, ch);
  const int64_t centre = n * down + half;                 // tap index of input frame j is centre - j*up
  int64_t j_lo = (centre - 2 * (int64_t)half + up - 1) / up;            // ceil((centre - 2 half) / up)
  if (centre - 2 * (int64_t)half < 0) j_lo = 0;
  int64_t j_hi = centre / up;                                            // floor
  if (j_hi > nframes - 1) j_hi = nframes - 1;
  double acc = 0.0;
  for (int64_t j = j_lo; j <= j_hi; ++j) acc += taps[centre - j * up] * (double)mono_at(pcm, fmt, j, ch);
  return (float)acc;
}

__global__ void __launch_bounds__(256) afp_pcm_frontend_kernel(const int16_t* pcm, int64_t nframes, int ch, int up,
                                                               int down, const double* taps, int half, float* out,
                                                               int64_t nout) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= nout) return;
  out[n] = frontend_sample(reinterpret_cast<const uint8_t*>(pcm), AFP_PCM_I16, nframes, ch, up, down, taps, half, n);
}

// One file of a batched front-end call, built on the host; nout = ceil(nframes * up / down).
struct PcmFileDesc : PcmFile {
  int64_t tap_off;      // first tap of the file's (up, down) design in the packed taps
  int32_t up, down, half;
};

__global__ void __launch_bounds__(256) afp_pcm_frontend_batch_kernel(const uint8_t* pcm, const PcmFileDesc* files,
                                                                     int nfiles, const double* taps, float* out) {
  const PcmFileDesc& f = files[pcm_block_file(files, nfiles)];
  const int64_t n = ((int64_t)blockIdx.x - f.block_base) * blockDim.x + threadIdx.x;
  const int64_t nout = f.nout;
  if (n >= nout) return;
  out[f.out_off + n] =
      frontend_sample(pcm + f.in_off, f.fmt, f.nframes, f.ch, f.up, f.down, taps + f.tap_off, f.half, n);
}

}  // namespace

extern "C" int afp_pcm_frontend(afp_ctx* c, const int16_t* pcm, int pcm_on_host, int64_t nframes, int32_t channels,
                                int32_t up, int32_t down, const double* taps, int32_t ntaps, float* out,
                                int out_on_host, int64_t* nout) {
  if (!c || nframes < 0 || channels < 1 || up < 1 || down < 1 || (nframes > 0 && (!pcm || !out)))
    return AFP_ERR_INVALID;
  const bool resample = !(up == 1 && down == 1);
  if (resample && (!taps || ntaps < 1 || !(ntaps & 1))) AFP_FAIL(c, AFP_ERR_INVALID, "taps: odd length required");
  AFP_CUDA(c, cudaSetDevice(c->device));
  const int64_t n_out = (nframes * up + down - 1) / down;                // ceil, as resample_poly
  if (nout) *nout = n_out;
  if (n_out == 0) return AFP_OK;
  const int16_t* dpcm = nullptr;
  double* dtaps = nullptr;
  float* dout = out;
  int rc;
  if ((rc = afp_stage(c, c->d_pcm_stage, pcm, (size_t)nframes * channels, pcm_on_host, &dpcm)) ||
      (rc = afp_carve(c, c->d_tmp, [&](Carver& k) {
         dtaps = resample ? k.take<double>(ntaps) : nullptr;
         if (out_on_host) dout = k.take<float>(n_out);
       })))
    return rc;
  if (resample) AFP_CUDA(c, afp_copy_in(c, dtaps, taps, (size_t)ntaps, 1));
  if ((rc = afp_launch(c, afp_pcm_frontend_kernel, (unsigned)((n_out + 255) / 256), 256, 0, dpcm, nframes, channels,
                       up, down, dtaps, (ntaps - 1) / 2, dout, n_out)))
    return rc;
  if (out_on_host) AFP_CUDA(c, afp_copy_out(c, out, dout, (size_t)n_out, 1));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  c->batch_valid = false;     // the PCM staging buffer of the last batch may have been reused
  return AFP_OK;
}

extern "C" int afp_pcm_frontend_batch_bytes(afp_ctx* c, const uint8_t* pcm, int pcm_on_host, int64_t pcm_bytes,
                                            int32_t nfiles, const int64_t* byte_offsets, const int32_t* formats,
                                            const int64_t* nframes, const int32_t* channels, const int32_t* up,
                                            const int32_t* down, int32_t npairs, const int32_t* pair_rates,
                                            const int64_t* tap_offsets, const double* taps, float* out,
                                            int64_t out_capacity, int64_t* out_offsets, int64_t* out_lengths) {
  if (!c) return AFP_ERR_INVALID;
  if (npairs < 0) AFP_FAIL(c, AFP_ERR_INVALID, "negative count");
  if (nfiles > 0 && (!up || !down)) AFP_FAIL(c, AFP_ERR_INVALID, "null per-file array");
  if (npairs > 0 && (!pair_rates || !tap_offsets || !taps)) AFP_FAIL(c, AFP_ERR_INVALID, "null taps table");
  // the taps table: one odd-length design per distinct (up, down), packed one after the other
  if (npairs > 0 && tap_offsets[0] != 0) AFP_FAIL(c, AFP_ERR_INVALID, "tap_offsets[0] must be 0");
  for (int p = 0; p < npairs; ++p) {
    const int64_t nt = tap_offsets[p + 1] - tap_offsets[p];
    if (pair_rates[2 * p] < 1 || pair_rates[2 * p + 1] < 1) AFP_FAIL(c, AFP_ERR_INVALID, "taps table: up and down must be >= 1");
    if (nt < 1 || !(nt & 1) || nt > INT32_MAX) AFP_FAIL(c, AFP_ERR_INVALID, "taps: odd length required");
  }
  std::vector<PcmFileDesc> d;
  int64_t blocks = 0;
  auto own = [&](int f, const std::string& tag, PcmFileDesc& x) -> int {
    x.up = up[f];
    x.down = down[f];
    if (x.up < 1 || x.down < 1) AFP_FAIL(c, AFP_ERR_INVALID, tag + "up and down must be >= 1");
    if (x.nframes > (INT64_MAX - x.down) / x.up) AFP_FAIL(c, AFP_ERR_INVALID, tag + "too long");
    if (!(x.up == 1 && x.down == 1)) {
      int p = 0;
      while (p < npairs && !(pair_rates[2 * p] == x.up && pair_rates[2 * p + 1] == x.down)) ++p;
      if (p == npairs) AFP_FAIL(c, AFP_ERR_INVALID, tag + "no taps for its (up, down)");
      x.tap_off = tap_offsets[p];
      x.half = (int32_t)((tap_offsets[p + 1] - tap_offsets[p] - 1) / 2);
    }
    x.nout = (x.nframes * x.up + x.down - 1) / x.down;                   // ceil, as resample_poly
    return AFP_OK;
  };
  const int rc = pcm_batch_layout(c, pcm, pcm_on_host, pcm_bytes, nfiles, byte_offsets, formats, nframes, channels, own,
                                  out, out_capacity, out_offsets, out_lengths, &d, &blocks);
  if (rc || !out || blocks == 0) return rc;                   // a refused call, a sizing call, or nothing to compute
  // every distinct design's taps go up once, after the descriptors
  return pcm_batch_launch(c, afp_pcm_frontend_batch_kernel, pcm, pcm_on_host, pcm_bytes, d, blocks,
                          {{taps, npairs > 0 ? tap_offsets[npairs] : 0}}, out);
}

extern "C" int afp_pcm_frontend_batch(afp_ctx* c, const int16_t* pcm, int pcm_on_host, int64_t pcm_len, int32_t nfiles,
                                      const int64_t* pcm_offsets, const int64_t* nframes, const int32_t* channels,
                                      const int32_t* up, const int32_t* down, int32_t npairs, const int32_t* pair_rates,
                                      const int64_t* tap_offsets, const double* taps, float* out, int64_t out_capacity,
                                      int64_t* out_offsets, int64_t* out_lengths) {
  if (!c) return AFP_ERR_INVALID;
  if (nfiles < 0 || pcm_len < 0 || pcm_len > INT64_MAX / 2) AFP_FAIL(c, AFP_ERR_INVALID, "negative count");
  if (nfiles > 0 && !pcm_offsets) AFP_FAIL(c, AFP_ERR_INVALID, "null per-file array");
  std::vector<int64_t> boff;
  std::vector<int32_t> fmt;
  pcm_i16_layout(nfiles, pcm_offsets, &boff, &fmt);
  return afp_pcm_frontend_batch_bytes(c, reinterpret_cast<const uint8_t*>(pcm), pcm_on_host, 2 * pcm_len, nfiles,
                                      boff.data(), fmt.data(), nframes, channels, up, down, npairs, pair_rates,
                                      tap_offsets, taps, out, out_capacity, out_offsets, out_lengths);
}
