// ffmpeg front-end on the device: interleaved int16 mono or stereo PCM -> the mono int16 stream
// `ffmpeg -i F -f s16le -ac 1 -ar 11025 -` writes for it (audio_read.py:196-203), scaled to float32
// v / 32768 as the reference's reader does.  libswresample (FFmpeg 8.0, library defaults) does:
//
//   equal rates   s16 arithmetic: stereo -> (16384 (l + r) + 16384) >> 15, mono as it is.
//   other rates   float32 arithmetic on x / 32768: each channel through a polyphase FIR of P phases
//                 x L taps (afp_swr_design), output n at input position n D / P (D = in / g,
//                 P = out / g <= 1024), summed as the library's x86 FMA3 kernel sums: eight lanes,
//                 lane k accumulating taps k, k+8, ... by fused multiply-add, then the lanes folded
//                 (k, k+4), (k, k+2), (0, 1).  Stereo: 0.5 l + 0.5 r of the two resampled channels.
//                 Then lrintf(v * 32768), clipped to int16.  Edges: the input is mirrored around its
//                 last sample for R samples and then around sample 0 (swr_edges).
//
// 24-bit, 32-bit and float input (afp_swr_frontend_batch_bytes) is read at the sample load
// (afp_pcm_formats.cuh) as the library reads it: at equal rates a mono file's samples become int16 directly
// (x >> 16, or the s16 rule of a float), and stereo is mixed in float32 as 0.5 l + 0.5 r of float(x) 2^-31
// or the float itself; other rates take those floats instead of x / 32768.  Outputs of float input at
// equal rates follow the library's buffers: its packed s16 rule, and its scalar rule for the file's last
// n % 16 frames (tests/wide_pcm_reference.py).
//
// tests/swr_reference.py states the same in NumPy; tests/test_ffmpeg_frontend_cpu.py holds it to the
// library's own output and tests/test_gpu_ffmpeg_frontend.py holds this kernel to both.  One thread
// computes one output and reads its taps from global memory through the cache.  A design has P L
// floats: 1 KB at 22050 Hz, 83 KB at 48000 Hz, up to 166 KB (32000 and 96000 Hz: 441 and 147 phases).
// tools/ffmpeg_frontend_timing.py measures the kernel against the default front-end.
//
// The batch's layout, checks, upload and launch are the default front-end's (afp_pcm_formats.cuh); here
// are only the geometry, the cached designs, the edges and swr_sample.  The package calls only the byte
// form; afp_swr_frontend_batch (int16) forwards to it for ABI callers.
#include <cmath>
#include <map>
#include <mutex>
#include <numeric>

#include "afp_internal.cuh"
#include "afp_pcm_formats.cuh"

namespace {

// 176400 Hz (528 taps) is held to the library; 192000 Hz (575 taps) is not yet, so longer designs are refused
constexpr int kFilterSize = 32, kPhaseCount = 1024, kLanes = 8, kMaxTaps = 528;
constexpr double kCutoff = 0.97, kBeta = 9.0;

struct SwrGeometry {
  int32_t P, D, L;
  double factor;
};

bool swr_geometry(int32_t in_rate, int32_t out_rate, SwrGeometry* g) {
  if (in_rate < 1 || out_rate < 1) return false;
  const int32_t d = std::gcd(in_rate, out_rate);
  g->P = out_rate / d;
  g->D = in_rate / d;
  if (g->P > kPhaseCount) return false;               // needs interpolated phases
  g->factor = std::min(out_rate * kCutoff / in_rate, 1.0);
  g->L = std::max((int32_t)std::ceil(kFilterSize / g->factor), 1);
  return g->L <= kMaxTaps;
}

double bessel_i0(double x) {  // power series, summed until the terms stop changing the sum
  double s = 1.0, t = 1.0;
  const double q = x * x / 4.0;
  for (int k = 1;; ++k) {
    t *= q / ((double)k * k);
    if (s + t == s) return s;
    s += t;
  }
}

void swr_design(const SwrGeometry& g, float* bank) {
  const int P = g.P, L = g.L, center = (L - 1) / 2;
  std::vector<double> tab((size_t)L);
  double norm = 0.0;
  const int nph = (P % 2) ? P : P / 2 + 1;
  for (int ph = 0; ph < nph; ++ph) {
    double s = g.factor == 1.0 ? std::sin(M_PI * ph / P) * ((center & 1) ? 1 : -1) : 0.0;
    for (int i = 0; i < L; ++i) {
      const double x = M_PI * ((double)(i - center) - (double)ph / P) * g.factor;
      double y = x == 0 ? 1.0 : (g.factor == 1.0 ? s / x : std::sin(x) / x);
      const double w = 2.0 * x / (g.factor * L * M_PI);
      y *= bessel_i0(kBeta * std::sqrt(std::max(1 - w * w, 0.0)));
      tab[i] = y;
      s = -s;
      if (ph == 0) norm += y;
    }
    for (int i = 0; i < L; ++i) bank[(size_t)ph * L + i] = (float)(tab[i] / norm);
    if (P % 2 == 0 && ph > 0)
      for (int i = 0; i < L; ++i) bank[(size_t)(P - ph) * L + L - 1 - i] = bank[(size_t)ph * L + i];
  }
}

// outputs for n input frames, as the library's buffering gives them: the end is mirrored for R samples
int64_t swr_edges(const SwrGeometry& g, int64_t n) {
  const int64_t P = g.P, D = g.D, L = g.L, S = (L - 1) / 2 + n;
  int64_t R;
  if (n <= L) {
    R = (n + 1) / 2;
    if (n + R <= L) return 0;
  } else {
    const int64_t made = ((S - L + 1) * P - 1) / D + 1;   // outputs before the end is reflected
    R = (std::min(S - made * D / P, L) + 1) / 2;
  }
  return ((S + R - L + 1) * P - 1) / D + 1;
}

// designs cached per (in, out) rate pair for the process
std::mutex g_design_mu;
std::map<std::pair<int32_t, int32_t>, std::vector<float>> g_designs;

const std::vector<float>& cached_design(int32_t in_rate, int32_t out_rate, const SwrGeometry& g) {
  std::lock_guard<std::mutex> lk(g_design_mu);
  auto& v = g_designs[{in_rate, out_rate}];
  if (v.empty()) {
    v.resize((size_t)g.P * g.L);
    swr_design(g, v.data());
  }
  return v;
}

struct SwrFileDesc : PcmFile {
  int64_t bank_off;
  int32_t P, D, L, resample;
};

// sample c of extended input position e: mirrored around the end, then around 0 (the output count keeps
// e within the reflected samples)
__device__ __forceinline__ float swr_in(const uint8_t* pcm, int fmt, int64_t n, int ch, int c, int64_t e) {
  if (e < 0) e = -e;
  if (e >= n) e = 2 * n - 1 - e;
  return pcm_f32(pcm, fmt, e * ch + c);
}

__device__ __forceinline__ float swr_channel(const uint8_t* pcm, const SwrFileDesc& f, const float* taps, int64_t start,
                                             int c) {
  float lane[kLanes];
#pragma unroll
  for (int k = 0; k < kLanes; ++k) lane[k] = 0.0f;
  for (int j = 0; j < f.L; j += kLanes) {
#pragma unroll
    for (int k = 0; k < kLanes; ++k)
      if (j + k < f.L) lane[k] = __fmaf_rn(swr_in(pcm, f.fmt, f.nframes, f.ch, c, start + j + k), __ldg(taps + j + k), lane[k]);
  }
  float a[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) a[k] = __fadd_rn(lane[k], lane[k + 4]);
  return __fadd_rn(__fadd_rn(a[0], a[2]), __fadd_rn(a[1], a[3]));
}

__device__ __forceinline__ float swr_sample(const uint8_t* pcm, const SwrFileDesc& f, const float* bank, int64_t n) {
  if (!f.resample) {
    int v;
    if (f.fmt == AFP_PCM_I16 && f.ch == 2) {
      const int16_t* p = reinterpret_cast<const int16_t*>(pcm);
      v = (16384 * ((int)p[2 * n] + (int)p[2 * n + 1]) + 16384) >> 15;
    } else if (f.fmt != AFP_PCM_F32 && f.ch == 1) {
      v = pcm_s16(pcm, f.fmt, n);
    } else {
      float m = pcm_f32(pcm, f.fmt, f.ch * n);
      if (f.ch == 2) m = __fadd_rn(__fmul_rn(m, 0.5f), __fmul_rn(pcm_f32(pcm, f.fmt, 2 * n + 1), 0.5f));
      // the library's buffers of float input are 4096-byte packets, a multiple of 16 frames
      v = n >= f.nframes - (f.nframes & 15) ? pcm_s16_scalar_rule(m) : pcm_s16_rule(m);
    }
    return (float)v * (1.0f / 32768.0f);
  }
  const int64_t k = n * f.D;
  const int64_t start = k / f.P - (f.L - 1) / 2;
  const float* taps = bank + (k % f.P) * f.L;
  float v = swr_channel(pcm, f, taps, start, 0);
  if (f.ch == 2) v = __fadd_rn(__fmul_rn(v, 0.5f), __fmul_rn(swr_channel(pcm, f, taps, start, 1), 0.5f));
  return (float)pcm_s16_rule(v) * (1.0f / 32768.0f);
}

__global__ void __launch_bounds__(256) afp_swr_frontend_kernel(const uint8_t* pcm, const SwrFileDesc* files, int nfiles,
                                                              const float* banks, float* out) {
  const SwrFileDesc f = files[pcm_block_file(files, nfiles)];
  const int64_t n = ((int64_t)blockIdx.x - f.block_base) * blockDim.x + threadIdx.x;
  if (n >= f.nout) return;
  out[f.out_off + n] = swr_sample(pcm + f.in_off, f, banks + f.bank_off, n);
}

}  // namespace

extern "C" int afp_swr_design(int32_t in_rate, int32_t out_rate, float* bank, int64_t capacity, int32_t* phases,
                              int32_t* taps) {
  SwrGeometry g;
  if (in_rate < 1 || out_rate < 1) return AFP_ERR_INVALID;
  if (!swr_geometry(in_rate, out_rate, &g)) return AFP_ERR_UNSUPPORTED;
  if (phases) *phases = g.P;
  if (taps) *taps = g.L;
  if (!bank) return AFP_OK;
  if (capacity < (int64_t)g.P * g.L) return AFP_ERR_INVALID;
  swr_design(g, bank);
  return AFP_OK;
}

extern "C" int afp_swr_length(int64_t nframes, int32_t in_rate, int32_t out_rate, int64_t* nout) {
  SwrGeometry g;
  if (nframes < 0 || in_rate < 1 || out_rate < 1 || !nout) return AFP_ERR_INVALID;
  if (in_rate == out_rate) {
    *nout = nframes;
    return AFP_OK;
  }
  if (!swr_geometry(in_rate, out_rate, &g)) return AFP_ERR_UNSUPPORTED;
  if (nframes > (INT64_MAX / 2 - g.L) / g.P) return AFP_ERR_INVALID;
  *nout = swr_edges(g, nframes);
  return AFP_OK;
}

extern "C" int afp_swr_frontend_batch_bytes(afp_ctx* c, const uint8_t* pcm, int pcm_on_host, int64_t pcm_bytes,
                                            int32_t nfiles, const int64_t* byte_offsets, const int32_t* formats,
                                            const int64_t* nframes, const int32_t* channels, const int32_t* rates,
                                            int32_t out_rate, float* out, int64_t out_capacity, int64_t* out_offsets,
                                            int64_t* out_lengths) {
  if (!c) return AFP_ERR_INVALID;
  if (out_rate < 1) AFP_FAIL(c, AFP_ERR_INVALID, "output rate must be >= 1");
  if (nfiles > 0 && !rates) AFP_FAIL(c, AFP_ERR_INVALID, "null per-file array");
  std::vector<SwrFileDesc> d;
  std::vector<int32_t> uniq;                               // distinct input rates, first use first
  std::vector<std::pair<const float*, int64_t>> banks;     // and their designs
  int64_t blocks = 0;
  auto own = [&](int f, const std::string& tag, SwrFileDesc& x) -> int {
    if (rates[f] < 1) AFP_FAIL(c, AFP_ERR_INVALID, tag + "sample rate must be >= 1");
    if (x.ch > 2) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, tag + "the ffmpeg front-end takes mono or stereo");
    x.resample = rates[f] != out_rate;
    x.P = x.D = x.L = 1;
    x.nout = x.nframes;
    if (!x.resample) return AFP_OK;
    SwrGeometry g;
    if (!swr_geometry(rates[f], out_rate, &g))
      AFP_FAIL(c, AFP_ERR_UNSUPPORTED, tag + std::to_string(rates[f]) + " Hz needs interpolated phases or more than 528 taps");
    if (x.nframes > (INT64_MAX / 2 - g.L) / g.P) AFP_FAIL(c, AFP_ERR_INVALID, tag + "too long");
    x.P = g.P;
    x.D = g.D;
    x.L = g.L;
    x.nout = swr_edges(g, x.nframes);
    size_t u = 0;
    while (u < uniq.size() && uniq[u] != rates[f]) x.bank_off += banks[u++].second;
    if (u == uniq.size()) {
      const std::vector<float>& bank = cached_design(rates[f], out_rate, g);
      uniq.push_back(rates[f]);
      banks.push_back({bank.data(), (int64_t)bank.size()});
    }
    return AFP_OK;
  };
  const int rc = pcm_batch_layout(c, pcm, pcm_on_host, pcm_bytes, nfiles, byte_offsets, formats, nframes, channels, own,
                                  out, out_capacity, out_offsets, out_lengths, &d, &blocks);
  if (rc || !out || blocks == 0) return rc;                   // a refused call, a sizing call, or nothing to compute
  // every distinct rate's design goes up once, after the descriptors
  return pcm_batch_launch(c, afp_swr_frontend_kernel, pcm, pcm_on_host, pcm_bytes, d, blocks, banks, out);
}

extern "C" int afp_swr_frontend_batch(afp_ctx* c, const int16_t* pcm, int pcm_on_host, int64_t pcm_len, int32_t nfiles,
                                      const int64_t* pcm_offsets, const int64_t* nframes, const int32_t* channels,
                                      const int32_t* rates, int32_t out_rate, float* out, int64_t out_capacity,
                                      int64_t* out_offsets, int64_t* out_lengths) {
  if (!c) return AFP_ERR_INVALID;
  if (nfiles < 0 || pcm_len < 0 || pcm_len > INT64_MAX / 2) AFP_FAIL(c, AFP_ERR_INVALID, "negative count");
  if (nfiles > 0 && !pcm_offsets) AFP_FAIL(c, AFP_ERR_INVALID, "null per-file array");
  std::vector<int64_t> boff;
  std::vector<int32_t> fmt;
  pcm_i16_layout(nfiles, pcm_offsets, &boff, &fmt);
  return afp_swr_frontend_batch_bytes(c, reinterpret_cast<const uint8_t*>(pcm), pcm_on_host, 2 * pcm_len, nfiles,
                                      boff.data(), fmt.data(), nframes, channels, rates, out_rate, out, out_capacity,
                                      out_offsets, out_lengths);
}
