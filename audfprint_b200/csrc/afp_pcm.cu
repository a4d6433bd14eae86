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
#include "afp_internal.cuh"

namespace {

__device__ __forceinline__ float mono_at(const int16_t* pcm, int64_t j, int ch) {
  const int16_t* p = pcm + j * ch;
  float s = 0.0f;
  for (int c = 0; c < ch; ++c) s += (float)p[c] * (1.0f / 32768.0f);
  return ch == 1 ? s : s / (float)ch;
}

__global__ void __launch_bounds__(256) afp_pcm_frontend_kernel(const int16_t* pcm, int64_t nframes, int ch, int up,
                                                               int down, const double* taps, int half, float* out,
                                                               int64_t nout) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= nout) return;
  if (up == 1 && down == 1) {
    out[n] = mono_at(pcm, n, ch);
    return;
  }
  const int64_t centre = n * down + half;                 // tap index of input frame j is centre - j*up
  int64_t j_lo = (centre - 2 * (int64_t)half + up - 1) / up;            // ceil((centre - 2 half) / up)
  if (centre - 2 * (int64_t)half < 0) j_lo = 0;
  int64_t j_hi = centre / up;                                            // floor
  if (j_hi > nframes - 1) j_hi = nframes - 1;
  double acc = 0.0;
  for (int64_t j = j_lo; j <= j_hi; ++j) acc += taps[centre - j * up] * (double)mono_at(pcm, j, ch);
  out[n] = (float)acc;
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
  const int16_t* dpcm = pcm;
  if (pcm_on_host) {
    AFP_CUDA(c, c->d_pcm_stage.reserve(sizeof(int16_t) * (size_t)nframes * channels + 16));
    AFP_CUDA(c, cudaMemcpyAsync(c->d_pcm_stage.p, pcm, sizeof(int16_t) * (size_t)nframes * channels,
                                cudaMemcpyHostToDevice, c->stream));
    dpcm = c->d_pcm_stage.as<int16_t>();
  }
  const double* dtaps = nullptr;
  if (resample) {
    AFP_CUDA(c, c->d_tmp.reserve(sizeof(double) * (size_t)ntaps + sizeof(float) * (size_t)(out_on_host ? n_out : 0) + 64));
    AFP_CUDA(c, cudaMemcpyAsync(c->d_tmp.p, taps, sizeof(double) * (size_t)ntaps, cudaMemcpyHostToDevice, c->stream));
    dtaps = c->d_tmp.as<double>();
  } else {
    AFP_CUDA(c, c->d_tmp.reserve(sizeof(float) * (size_t)(out_on_host ? n_out : 0) + 64));
  }
  float* dout = out;
  if (out_on_host) dout = reinterpret_cast<float*>(c->d_tmp.as<char>() + (resample ? ((sizeof(double) * (size_t)ntaps + 15) & ~(size_t)15) : 0));
  afp_pcm_frontend_kernel<<<(unsigned)((n_out + 255) / 256), 256, 0, c->stream>>>(dpcm, nframes, channels, up, down,
                                                                                 dtaps, (ntaps - 1) / 2, dout, n_out);
  AFP_CUDA(c, cudaGetLastError());
  c->launches++;
  if (out_on_host)
    AFP_CUDA(c, cudaMemcpyAsync(out, dout, sizeof(float) * (size_t)n_out, cudaMemcpyDeviceToHost, c->stream));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  c->batch_valid = false;     // the PCM staging buffer of the last batch may have been reused
  return AFP_OK;
}
