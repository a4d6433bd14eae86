// K1 — fused framing + Hann window + 512-point real FFT + log-magnitude (FP64).
//
// Replaces stft.stft (reference stft.py:62-94: reflect pad 256, hop-256
// framing, window multiply, rfft) and the |.| / log part of
// Analyzer.find_peaks (audfprint_analyze.py:280-285).  The two whole-file
// reductions that follow (floor = max/1e6, mean, :283-286) are produced as
// per-tile partials here and finished in afp_stats_kernel; the per-bin high-pass
// (:293-295) is a time recursion and lives in the peak kernel (afp_peaks.cu).
//
// Work decomposition: a tile = 16 consecutive frames of one item (file x shift).
// PERSISTENT CTAs (2 per SM) walk the tile list; the hop-strided PCM of a tile
// is ONE contiguous run of 17*256 samples, staged into a double-buffered shared
// memory ring by 1-D TMA bulk copies (cp.async.bulk + mbarrier) issued one tile
// ahead, so the copy of tile i+1 overlaps the FFTs of tile i (edge tiles and
// unaligned files take a reflected scalar-load path).  16 threads cooperate on
// a frame: 256-point complex FFT as 16 x 16 with one padded shared-memory
// transpose, then the real-FFT split done on (k, 256-k) PAIRS so that each
// partner exchange (warp shuffle) and each W512 twiddle serves two bins.
//
// Why FP64: the peak decisions downstream compare these values bit-for-bit the
// way the reference's float64 NumPy path does; an FP32 spectrogram flips a
// decision roughly once per 10^5 frames (DESIGN.md "Precision").  The kernel is
// therefore bound by the FP64 pipe (64 lanes/clk/SM), not by HBM; the log is a
// table-driven FP64 routine (10 FP64 ops instead of libdevice's ~30).  The opt-in
// FP32 spectrogram mode is the same kernel over R = float; K1Traits<R> holds what
// differs between the two precisions.
#include <math.h>
#include <algorithm>
#include "afp_fft.cuh"
#include "afp_internal.cuh"
#include "afp_tma.cuh"

namespace {

constexpr int FT = AFP_FRAMES_PER_TILE;   // 16 frames per tile
constexpr int XS = 17;                    // padded row stride of the 16x16 exchange
constexpr int XF = 16 * XS;               // 272 values per frame per component
constexpr int K1_THREADS = 256;
constexpr int LOGTAB = 64;                // log table entries (6 mantissa bits) ...
constexpr int LOGCOPIES = 8;              // ... each stored 8 times, copy j in the 16-byte bank group j:
                                          // lane (l & 7) reads copy (l & 7), so the random lookups of a
                                          // quarter-warp never collide (4 wavefronts per LDS.128, always)

// np.pad(..., mode='reflect') index map (edge sample not repeated), any number
// of bounces (stft.py:88; SURVEY.md A.1).
__device__ __forceinline__ int64_t reflect_index(int64_t j, int64_t n) {
  if (n == 1) return 0;
  const int64_t period = 2 * (n - 1);
  int64_t r = j % period;
  if (r < 0) r += period;
  return r < n ? r : period - r;
}

// exact small-int -> double without the (slow) I2F.F64 path: (1.5*2^52 + x) - 1.5*2^52
__device__ __forceinline__ double int_to_double(int x) {
  return __hiloint2double(0x43380000 + (x >> 31), x) - 6755399441055744.0;
}

// 0.5*log(0.25*v) for v > 0 normal; table-driven, |abs error| ~ 1e-16 + 0.5 ulp.
//   v = 2^e * m, m in [1,2); i = top 6 mantissa bits; r = m*c_i - 1, |r| <= 2^-7
//   0.5*log(v/4) = (e-2)*ln2/2 + t_i + 0.5*log1p(r),  t_i = -0.5*log(c_i)
// Inputs that are 0 / denormal / inf / nan give a meaningless value here; the
// caller detects them with is_special() and patches with half_log_quarter_slow().
__device__ __noinline__ double half_log_quarter_slow(double v) { return 0.5 * log(0.25 * v); }
__device__ __forceinline__ bool is_special(double v) {
  return (unsigned)(__double2hiint(v) - 0x00100000) >= 0x7fe00000u;
}

// The coefficients of 0.5*log1p(r) and ln2/2.  They live in constant memory so that the DFMAs
// take them as c[][] operands: as literals, every one without a zero low word is rebuilt in
// registers at each of the nine inlined log call sites.
__constant__ double k1_log_c64[8] = {0.5 / 7.0, -0.5 / 6.0, 0.5 / 5.0, -0.5 / 4.0,
                                     0.5 / 3.0, -0.5 / 2.0, 0.5,       0.34657359027997264};

// s_logtab_lane = table base + (lane & 7): this lane's private copy (stride LOGCOPIES).
__device__ __forceinline__ double half_log_quarter(double v, const double2* s_logtab_lane) {
  const int hi = __double2hiint(v);
  const int lo = __double2loint(v);
  const double m = __hiloint2double((hi & 0x000fffff) | 0x3ff00000, lo);
  const double2 ct = s_logtab_lane[((hi >> 14) & (LOGTAB - 1)) * LOGCOPIES];
  const double r = fma(m, ct.x, -1.0);
  double p = k1_log_c64[0];
  p = fma(p, r, k1_log_c64[1]);
  p = fma(p, r, k1_log_c64[2]);
  p = fma(p, r, k1_log_c64[3]);
  p = fma(p, r, k1_log_c64[4]);
  p = fma(p, r, k1_log_c64[5]);
  p = fma(p, r, k1_log_c64[6]);
  const double ed = int_to_double((hi >> 20) - 1025);
  return fma(ed, k1_log_c64[7], ct.y) + p * r;   // ln2/2
}

template <typename PcmT> struct PcmTraits;
template <> struct PcmTraits<int16_t> {
  static constexpr int NBUF = 2;
};
template <> struct PcmTraits<float> {
  static constexpr int NBUF = 1;   // 2 x 17 KB would not leave room for two CTAs per SM
};

// What differs between the two spectrogram precisions of K1.  load2 converts two PCM samples
// (int16 unscaled: the window carries the 2^-15); log_pair / log1 give 0.5*log(0.25*v) of
// v = 4|X|^2; hbits maps a positive v to an int that orders like it, HMIN_NONE being the value
// of a warp without a frame; log_lower_bound turns the warp's minimum hbits into a lower bound
// of its smallest log.
template <typename R> struct K1Traits;

// FP64 (default): table-driven log, bit-exact downstream.
template <> struct K1Traits<double> {
  using R2 = double2;
  static constexpr int MIN_CTAS = 2;                    // per SM: 2 x 256 threads x <= 128 registers
  static constexpr int LOGTAB_N = LOGTAB * LOGCOPIES;   // log table entries staged in shared memory
  static constexpr int HMIN_NONE = 0x7ff00000;          // high word of +inf
  __device__ static __forceinline__ void load2(const int16_t* p, double& a, double& b) {
    const uint32_t w = *reinterpret_cast<const uint32_t*>(p);
    a = int_to_double((int)(short)(w & 0xffffu));
    b = int_to_double((int)w >> 16);
  }
  __device__ static __forceinline__ void load2(const float* p, double& a, double& b) {
    const float2 w = *reinterpret_cast<const float2*>(p);
    a = (double)w.x;
    b = (double)w.y;
  }
  // the high word alone: positive doubles order like their bits
  __device__ static __forceinline__ int hbits(double v) { return __double2hiint(v); }
  __device__ static __forceinline__ void log_pair(double ssa, double ssb, const double2* tab, double& la,
                                                  double& lb) {
    la = half_log_quarter(ssa, tab);
    lb = half_log_quarter(ssb, tab);
    if (is_special(ssa) || is_special(ssb)) {   // digital silence etc.: rare, off the hot path
      la = half_log_quarter_slow(ssa);
      lb = half_log_quarter_slow(ssb);
    }
  }
  __device__ static __forceinline__ double log1(double ss, const double2* tab) {
    double lg = half_log_quarter(ss, tab);
    if (is_special(ss)) lg = half_log_quarter_slow(ss);
    return lg;
  }
  // the log of the high word with the low word zeroed: the statistics pass only asks "is
  // anything below the floor?"; a false alarm just takes its exact path
  __device__ static __forceinline__ double log_lower_bound(int hmin, const double2* tab) {
    const double v_lo = __hiloint2double(hmin, 0);
    return hmin >= HMIN_NONE ? INFINITY : (hmin < 0x00100000 ? -INFINITY : half_log_quarter(v_lo, tab));
  }
};

// FP32 (Analyzer.precision = 'fp32', opt-in): FFT, |.|^2 and log (MUFU) in single precision,
// float log-spectrogram out: half the output bytes, twice the FP32 lane rate, ~80 registers ->
// three CTAs per SM.  Downstream decisions then see values that differ from the reference's
// by ~1e-7 relative, so hashes are NOT guaranteed bit-identical (measured in bench.py).
template <> struct K1Traits<float> {
  using R2 = float2;
  static constexpr int MIN_CTAS = 3;                    // per SM: 3 x 256 threads x <= 80 registers
  static constexpr int LOGTAB_N = 0;
  static constexpr int HMIN_NONE = 0x7f800000;          // bits of +inf
  __device__ static __forceinline__ void load2(const int16_t* p, float& a, float& b) {
    const uint32_t w = *reinterpret_cast<const uint32_t*>(p);
    a = (float)(short)(w & 0xffffu);
    b = (float)((int)w >> 16);
  }
  __device__ static __forceinline__ void load2(const float* p, float& a, float& b) {
    const float2 w = *reinterpret_cast<const float2*>(p);
    a = w.x;
    b = w.y;
  }
  __device__ static __forceinline__ int hbits(float v) { return __float_as_int(v); }
  __device__ static __forceinline__ void log_pair(float ssa, float ssb, const double2*, float& la, float& lb) {
    la = 0.5f * __logf(0.25f * ssa);
    lb = 0.5f * __logf(0.25f * ssb);
  }
  __device__ static __forceinline__ float log1(float ss, const double2*) { return 0.5f * __logf(0.25f * ss); }
  // the exact minimum's log, less a margin for __logf's error so that it stays a lower bound
  __device__ static __forceinline__ double log_lower_bound(int hmin, const double2*) {
    return hmin >= HMIN_NONE ? INFINITY
           : (hmin < 0x00800000 ? -INFINITY : (double)(0.5f * __logf(0.25f * __int_as_float(hmin))) - 1e-6);
  }
};

template <typename R>
struct StftArgs {
  using R2 = typename K1Traits<R>::R2;
  const void* pcm;
  const ItemDesc* items;
  const int32_t* tile_item;   // [ntiles] item of every tile (built by afp_tile_table_kernel)
  int nitems;
  int tile_begin, tile_end;   // tile range of this launch (a chunk of the batch)
  const R* window;        // 512 (pre-scaled by 2^-15 for int16 PCM)
  const R2* tw256;        // [p][r] = W256^(r*p), (cos, -sin)
  const R2* w512;         // 256: (cos, -sin)(2 pi k / 512)
  const double2* logtab;  // [64][8]: (c_i, -0.5*log(c_i)), 8 identical copies interleaved (FP64 only)
  R* logs;                // [frames][256]
  double* nyq;            // [frames]
  double* tile_stats;     // [tiles][3]
  double* mag;            // optional [frames][257]
};

struct TileInfo {
  int64_t frame0;     // batch-wide index of the tile's first frame
  int64_t src;        // absolute sample index of the run's first sample (sample_start + j0)
  int64_t j0;         // the same relative to the item (may be < 0)
  int64_t nsamples;   // samples of the item (reflection period)
  int nft;            // frames of the tile that exist
  int tma;            // (first << 16) | count: samples [first, first+count) of the run come by one bulk
                      // copy (count == 0: none); whatever else the run holds - the reflected head of a
                      // file's first tile, the tail of its last - is staged by scalar loads
};

template <typename PcmT>
__device__ __forceinline__ TileInfo make_tile(const PcmT* pcm, const ItemDesc& it, int tile) {
  TileInfo ti;
  const int t0 = (tile - it.tile_base) * FT;
  ti.frame0 = it.frame_base + t0;
  ti.nft = min(FT, it.nframes - t0);
  ti.j0 = (int64_t)(t0 - 1) * AFP_N_HOP;   // first sample of the run (may be < 0)
  ti.src = it.sample_start + ti.j0;
  ti.nsamples = it.nsamples;
  // the part of the run that lies inside the file, trimmed to 16-byte granules; the shared-memory
  // buffer is 16-byte aligned, so source and destination agree iff the run itself starts on one
  constexpr int GR = 16 / (int)sizeof(PcmT);
  const int64_t run_n = (int64_t)(ti.nft + 1) * AFP_N_HOP;
  const int64_t lo = ti.j0 < 0 ? -ti.j0 : 0;
  const int64_t hi = (ti.j0 + run_n <= it.nsamples ? run_n : it.nsamples - ti.j0) & ~(int64_t)(GR - 1);
  const bool aligned = (reinterpret_cast<uintptr_t>(pcm + ti.src) & 15) == 0;
  ti.tma = (aligned && hi > lo) ? (int)((lo << 16) | (hi - lo)) : 0;   // lo is 0 or 256: a granule multiple
  return ti;
}

// Stage the PCM run of a tile: TMA bulk copy (one thread) or reflected loads (all).
template <typename PcmT>
__device__ __forceinline__ void stage_tile(const PcmT* pcm, const TileInfo& ti, PcmT* dst, unsigned long long* bar) {
  const int nsamp = (ti.nft + 1) * AFP_N_HOP;
  const int t_first = ti.tma >> 16, t_count = ti.tma & 0xffff;
  if (t_count && threadIdx.x == 0) bulk_copy_g2s(dst + t_first, pcm + ti.src + t_first, t_count * sizeof(PcmT), bar);
  if (t_count != nsamp) {   // samples outside the bulk copy: [0, t_first) and [t_first + t_count, nsamp)
    const PcmT* item0 = pcm + (ti.src - ti.j0);
    for (int i = threadIdx.x; i < nsamp - t_count; i += K1_THREADS) {
      const int p = i < t_first ? i : i + t_count;
      dst[p] = item0[reflect_index(ti.j0 + p, ti.nsamples)];
    }
  }
}

// Shared memory of one K1 CTA; the kernel carves it up in this order.
template <typename R, typename PcmT>
constexpr size_t k1_smem_bytes() {
  return 512 * sizeof(R) + 2 * 256 * sizeof(typename K1Traits<R>::R2) + K1Traits<R>::LOGTAB_N * sizeof(double2) +
         2 * FT * XF * sizeof(R) + 2 * 24 * sizeof(double) + 2 * sizeof(unsigned long long) +
         PcmTraits<PcmT>::NBUF * (FT + 1) * AFP_N_HOP * sizeof(PcmT);
}

// `a` is __grid_constant__: its fields are read from the parameter bank where they are used.
// Passed by value, a struct this small is copied into registers at entry, and its pointers
// then stay live across the whole persistent loop and spill.
template <typename R, typename PcmT, bool WRITE_MAG>
__global__ void __launch_bounds__(K1_THREADS, K1Traits<R>::MIN_CTAS)
    afp_stft_kernel(const __grid_constant__ StftArgs<R> a) {
  using Tr = K1Traits<R>;
  using R2 = typename Tr::R2;
  constexpr int NBUF = PcmTraits<PcmT>::NBUF;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  R* s_win = reinterpret_cast<R*>(smem_raw);                           // 512
  R2* s_tw256 = reinterpret_cast<R2*>(s_win + 512);                    // 256, [p][r]
  R2* s_w512 = s_tw256 + 256;                                          // 256
  double2* s_logtab_all = reinterpret_cast<double2*>(s_w512 + 256);    // Tr::LOGTAB_N
  R* s_xr = reinterpret_cast<R*>(s_logtab_all + Tr::LOGTAB_N);         // FT * XF
  R* s_xi = s_xr + FT * XF;                                            // FT * XF
  double* s_red = reinterpret_cast<double*>(s_xi + FT * XF);           // 2 x 3 * 8
  unsigned long long* s_bar = reinterpret_cast<unsigned long long*>(s_red + 2 * 24);   // 2
  PcmT* s_pcm = reinterpret_cast<PcmT*>(s_bar + 2);                    // NBUF * (FT+1)*256, 16 B aligned
  constexpr int PCM_BUF = (FT + 1) * AFP_N_HOP;
  const PcmT* pcm = reinterpret_cast<const PcmT*>(a.pcm);

  const int tid = threadIdx.x;
  if (tid == 0) mbar_init<2>(s_bar);
  for (int i = tid; i < 512; i += K1_THREADS) s_win[i] = a.window[i];
  for (int i = tid; i < 256; i += K1_THREADS) {
    s_tw256[i] = a.tw256[i];
    s_w512[i] = a.w512[i];
  }
  if constexpr (Tr::LOGTAB_N > 0)
    for (int i = tid; i < Tr::LOGTAB_N; i += K1_THREADS) s_logtab_all[i] = a.logtab[i];
  __syncthreads();

  const int g = tid >> 4;   // frame within the tile
  const int r = tid & 15;   // cooperating thread within the frame
  const int lane = tid & 31;
  const double2* s_logtab = s_logtab_all + (lane & (LOGCOPIES - 1));   // this lane's copy of the log table
  const int src_lane = (lane & 16) | ((16 - r) & 15);
  uint32_t phases = 0u;   // bit b = parity to wait for on barrier b

  int tile = a.tile_begin + blockIdx.x;
  if (tile >= a.tile_end) return;
  const int G = gridDim.x;
  // Tile descriptors are fetched two tiles ahead so that their (dependent) global
  // loads never sit on the critical path: item index at distance 3, ItemDesc at 2.
  TileInfo cur = make_tile(pcm, a.items[a.tile_item[tile]], tile);
  TileInfo nxt = cur;
  if (tile + G < a.tile_end) nxt = make_tile(pcm, a.items[a.tile_item[tile + G]], tile + G);
  int item_nn = (tile + 2 * G < a.tile_end) ? a.tile_item[tile + 2 * G] : 0;
  stage_tile(pcm, cur, s_pcm, s_bar);
  int buf = 0;
  int red = 0;   // NBUF == 1: which half of s_red this iteration's partials go to (NBUF == 2: buf)

  for (; tile < a.tile_end; tile += G) {
    const int next = tile + G;
    // prefetch the next tile into the other buffer (free since the end-of-iteration barrier)
    if (NBUF == 2 && next < a.tile_end) stage_tile(pcm, nxt, s_pcm + (buf ^ 1) * PCM_BUF, s_bar + (buf ^ 1));
    ItemDesc desc_nn = a.items[item_nn];                                   // consumed at the end of the iteration
    const int item_n3 = (tile + 3 * G < a.tile_end) ? a.tile_item[tile + 3 * G] : 0;   // consumed next iteration
    if (cur.tma & 0xffff) {
      mbar_wait(s_bar + buf, (phases >> buf) & 1u);
      phases ^= 1u << buf;
    }
    if ((cur.tma & 0xffff) != (cur.nft + 1) * AFP_N_HOP) __syncthreads();   // scalar-staged samples are visible

    const bool active = g < cur.nft;
    const int64_t frame = cur.frame0 + g;
    R vmax = 0, vsum = 0;
    int hmin = Tr::HMIN_NONE;   // min of hbits(4|X|^2)
    R zr[16], zi[16];
    if (active) {
      // step A: z[16q + r] = (x[2n] w[2n], x[2n+1] w[2n+1]), n = 16q + r
      const PcmT* fr = s_pcm + buf * PCM_BUF + g * AFP_N_HOP;
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        const int i0 = 2 * (16 * q + r);
        const R2 w = *reinterpret_cast<const R2*>(s_win + i0);
        R x0, x1;
        Tr::load2(fr + i0, x0, x1);
        zr[q] = x0 * w.x;
        zi[q] = x1 * w.y;
      }
      afp_fft16(zr, zi);
      R* xr = s_xr + g * XF;
      R* xi = s_xi + g * XF;
#pragma unroll
      for (int p = 0; p < 16; ++p) {
        const R2 w = s_tw256[p * 16 + r];
        xr[p * XS + r] = zr[p] * w.x - zi[p] * w.y;
        xi[p * XS + r] = zr[p] * w.y + zi[p] * w.x;
      }
    }
    __syncwarp();
    if (active) {
      // step B: thread p = r transforms column p: Z[p + 16 s]
      const R* xr = s_xr + g * XF + r * XS;
      const R* xi = s_xi + g * XF + r * XS;
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        zr[q] = xr[q];
        zi[q] = xi[q];
      }
      afp_fft16(zr, zi);
    }
    // real-FFT split on pairs (k, 256-k), k = r + 16 s, s < 8: the partner
    // Z[(256-k)&255] sits in lane (16-r)&15, register 15-s (r > 0) or (16-s)&15 (r == 0).
    //   2Xe = Z[k] + conj(Zp), 2Xo = -i (Z[k] - conj(Zp)), P = W512^k * 2Xo
    //   4|X[k]|^2 = |2Xe + P|^2,  4|X[256-k]|^2 = |2Xe - P|^2
    {
      R* out = a.logs + frame * AFP_NBINS;
#pragma unroll
      for (int s = 0; s < 8; ++s) {
        R c = __shfl_sync(0xffffffffu, zr[15 - s], src_lane);
        R d = __shfl_sync(0xffffffffu, zi[15 - s], src_lane);
        if (r == 0) {
          c = zr[(16 - s) & 15];
          d = zi[(16 - s) & 15];
        }
        if (active) {
          const int k = r + 16 * s;
          const R2 w = s_w512[k];
          const R er = zr[s] + c, ei = zi[s] - d, orr = zi[s] + d, oi = c - zr[s];
          const R pr = w.x * orr - w.y * oi, pi = w.x * oi + w.y * orr;
          const R ar = er + pr, ai = ei + pi, br = er - pr, bi = ei - pi;
          const R ssa = ar * ar + ai * ai;   // 4 |X[k]|^2
          const R ssb = br * br + bi * bi;   // 4 |X[256-k]|^2
          R la, lb;
          Tr::log_pair(ssa, ssb, s_logtab, la, lb);
          out[k] = la;
          if (k != 0) out[256 - k] = lb; else a.nyq[frame] = lb;   // k == 0 pairs with the Nyquist bin
          if (WRITE_MAG) {
            a.mag[frame * 257 + k] = sqrt(R(0.25) * ssa);
            a.mag[frame * 257 + 256 - k] = sqrt(R(0.25) * ssb);
          }
          vmax = fmax(vmax, fmax(ssa, ssb));
          hmin = min(hmin, min(Tr::hbits(ssa), Tr::hbits(ssb)));
          vsum += la + lb;
        }
      }
      if (active && r == 0) {   // bin 128 pairs with itself
        const R2 w = s_w512[128];
        const R er = R(2) * zr[8], orr = R(2) * zi[8];   // ei = 0, oi = 0
        const R ar = er + w.x * orr, ai = w.y * orr;
        const R ss = ar * ar + ai * ai;
        const R lg = Tr::log1(ss, s_logtab);
        out[128] = lg;
        if (WRITE_MAG) a.mag[frame * 257 + 128] = sqrt(R(0.25) * ss);
        vmax = fmax(vmax, ss);
        hmin = min(hmin, Tr::hbits(ss));
        vsum += lg;
      }
    }
    // deterministic CTA reduction of (max |S|^2, min log, sum log), in FP64 for both precisions.
    // The partials alternate between the two halves of s_red: thread 0 reads this tile's half after
    // the barrier below, and when the next tile is wholly bulk-copied no barrier comes before the
    // other warps write their next partials.  They go to the other half; writing this half again
    // needs the next iteration's barrier, which thread 0 reaches only once it has read.
    hmin = __reduce_min_sync(0xffffffffu, hmin);
    const double vmin = Tr::log_lower_bound(hmin, s_logtab);   // +inf: this warp had no frame in the tile
    double dmax = vmax, dsum = vsum;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      dmax = fmax(dmax, __shfl_xor_sync(0xffffffffu, dmax, o));
      dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
    }
    double* const s_part = s_red + 24 * (NBUF == 2 ? buf : red);
    if (lane == 0) {
      s_part[(tid >> 5) * 3 + 0] = dmax;
      s_part[(tid >> 5) * 3 + 1] = vmin;
      s_part[(tid >> 5) * 3 + 2] = dsum;
    }
    __syncthreads();   // also: every thread is done with s_pcm[buf]
    if (tid == 0) {
      double m = 0.0, mn = INFINITY, sm = 0.0;
#pragma unroll
      for (int w = 0; w < K1_THREADS / 32; ++w) {
        m = fmax(m, s_part[w * 3 + 0]);
        mn = fmin(mn, s_part[w * 3 + 1]);
        sm += s_part[w * 3 + 2];
      }
      a.tile_stats[(size_t)tile * 3 + 0] = 0.25 * m;
      a.tile_stats[(size_t)tile * 3 + 1] = mn;
      a.tile_stats[(size_t)tile * 3 + 2] = sm;
    }
    if (NBUF == 2) buf ^= 1; else red ^= 1;
    cur = nxt;
    if (tile + 2 * G < a.tile_end) nxt = make_tile(pcm, desc_nn, tile + 2 * G);
    item_nn = item_n3;
    if (NBUF == 1 && next < a.tile_end) stage_tile(pcm, cur, s_pcm, s_bar);
  }
}

// tile -> item table (one thread per item)
__global__ void afp_tile_table_kernel(const ItemDesc* items, int nitems, int32_t* tile_item) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nitems) return;
  const ItemDesc it = items[i];
  const int nt = (it.nframes + FT - 1) / FT;
  for (int k = 0; k < nt; ++k) tile_item[it.tile_base + k] = i;
}

// ---- per-item statistics: floor, mean (audfprint_analyze.py:283-286) ----------
// Three tiny launches.  (1) one WARP per item reduces the tile partials in a fixed order
// (deterministic): floor, all-zero flag, mean of the un-floored logs, and whether anything
// may sit below the floor.  (2) For such items only (digital silence, or the rare file whose
// smallest bin is 120 dB below its largest) the tile sums are recomputed with the floor
// applied, one CTA per tile so that a single long file cannot serialise the batch.
// (3) the means of those items are re-reduced.
__global__ void __launch_bounds__(256) afp_stats_kernel(const ItemDesc* items, int item0, int nitems,
                                                        const double* tile_stats, ItemStats* out, int phase) {
  const int lane = threadIdx.x & 31;
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= nitems) return;
  const int item = item0 + w;
  if (phase == 1 && !out[item].floored) return;       // only items whose tile sums were floored
  const ItemDesc it = items[item];
  const int ntiles = (it.nframes + FT - 1) / FT;
  double m = 0.0, mn = INFINITY, sm = 0.0;
  for (int i = lane; i < ntiles; i += 32) {
    const double* ts = tile_stats + (size_t)(it.tile_base + i) * 3;
    m = fmax(m, ts[0]);
    mn = fmin(mn, ts[1]);
    sm += ts[2];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    sm += __shfl_xor_sync(0xffffffffu, sm, o);
  }
  if (lane == 0) {
    const bool allzero = !(m > 0.0);
    ItemStats st;
    st.logfloor = allzero ? 0.0 : log(sqrt(m) / 1e6);
    st.mean = (allzero || it.nframes == 0) ? 0.0 : sm / ((double)it.nframes * 257.0);
    st.allzero = allzero ? 1 : 0;
    st.floored = (phase == 0 && !allzero && mn < st.logfloor) ? 1 : 0;   // needs the floored sums
    out[item] = st;
  }
}

// floored tile sums of the flagged items: grid (items, FS_SPLIT); un-flagged items leave after
// one load, a flagged item's tiles are dealt round-robin to its FS_SPLIT CTAs
constexpr int FS_SPLIT = 8;
template <typename R>
__global__ void __launch_bounds__(256) afp_floorsum_kernel(const ItemDesc* items, int item0, const ItemStats* stats,
                                                           const R* logs, const double* nyq,
                                                           double* tile_stats) {
  __shared__ double s_part[8];
  const int item = item0 + blockIdx.x;
  const ItemStats st = stats[item];
  if (!st.floored) return;                        // uniform
  const ItemDesc it = items[item];
  const int ntiles = (it.nframes + FT - 1) / FT;
  for (int k = blockIdx.y; k < ntiles; k += FS_SPLIT) {
    const int t0 = k * FT, nft = min(FT, it.nframes - t0);
    const R* L = logs + (size_t)(it.frame_base + t0) * AFP_NBINS;
    double acc = 0.0;
    for (int i = threadIdx.x; i < nft * AFP_NBINS; i += 256) acc += fmax((double)L[i], st.logfloor);
    if ((int)threadIdx.x < nft) acc += fmax(nyq[it.frame_base + t0 + threadIdx.x], st.logfloor);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < 8; ++w) t += s_part[w];
      tile_stats[(size_t)(it.tile_base + k) * 3 + 2] = t;
    }
  }
}

// ---- conditioned spectrogram for the parity entry point afp_sgram -------------
// One thread per (item, bin); serial over time.  Not on the product path (the
// peak kernel fuses this recursion); exists so that the test can compare the
// sgram itself with the oracle.
template <typename R>
__global__ void afp_sgram_kernel(const ItemDesc* items, const ItemStats* stats, const R* logs,
                                 double pole, double* out) {
  const ItemDesc it = items[blockIdx.x];
  const ItemStats st = stats[blockIdx.x];
  const int b = threadIdx.x;
  double z = 0.0;
  for (int t = 0; t < it.nframes; ++t) {
    const size_t idx = (size_t)(it.frame_base + t) * AFP_NBINS + b;
    double x = st.allzero ? 0.0 : __dsub_rn(fmax((double)logs[idx], st.logfloor), st.mean);
    const double y = __dadd_rn(z, x);
    z = __dadd_rn(-x, __dmul_rn(pole, y));
    out[idx] = y;
  }
}

}  // namespace

int afp_launch_tile_table(afp_ctx* c) {
  if (c->nitems == 0) return AFP_OK;
  afp_tile_table_kernel<<<(c->nitems + 255) / 256, 256, 0, c->stream>>>(c->d_items.as<ItemDesc>(), c->nitems,
                                                                       c->d_tile_item.as<int32_t>());
  AFP_CUDA(c, cudaGetLastError());
  c->launches++;
  return AFP_OK;
}

namespace {

// One K1 instantiation: num_sms x its CTAs per SM, at most one CTA per tile.
template <typename R, typename PcmT, bool WRITE_MAG>
cudaError_t launch_k1(const StftArgs<R>& a, int num_sms, int64_t ntiles, cudaStream_t stream) {
  constexpr size_t smem = k1_smem_bytes<R, PcmT>();
  const int nctas = (int)std::min<int64_t>(ntiles, (int64_t)num_sms * K1Traits<R>::MIN_CTAS);
  const cudaError_t e =
      cudaFuncSetAttribute(afp_stft_kernel<R, PcmT, WRITE_MAG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e == cudaSuccess) afp_stft_kernel<R, PcmT, WRITE_MAG><<<nctas, K1_THREADS, smem, stream>>>(a);
  return e;
}

// window: 2 x 512 (the second pre-scaled by 2^-15 for int16 PCM); twid: tw256, then W512
template <typename R>
cudaError_t launch_stft(afp_ctx* c, const DevBuf& window, const DevBuf& twid, const void* pcm, int dtype,
                        double* mag_out, int64_t tile0, int64_t ntiles) {
  using R2 = typename K1Traits<R>::R2;
  StftArgs<R> a;
  a.pcm = pcm;
  a.items = c->d_items.as<ItemDesc>();
  a.tile_item = c->d_tile_item.as<int32_t>();
  a.nitems = c->nitems;
  a.tile_begin = (int)tile0;
  a.tile_end = (int)(tile0 + ntiles);
  a.window = window.as<R>() + (dtype == AFP_PCM_I16 ? AFP_N_FFT : 0);
  a.tw256 = twid.as<R2>();
  a.w512 = twid.as<R2>() + 256;
  a.logtab = c->d_twid.as<double2>() + 512;
  a.logs = c->d_logs.as<R>();
  a.nyq = c->d_nyq.as<double>();
  a.tile_stats = c->d_tile_stats.as<double>();
  a.mag = mag_out;
  const int n = c->num_sms;
  if (dtype == AFP_PCM_I16)
    return mag_out ? launch_k1<R, int16_t, true>(a, n, ntiles, c->stream)
                   : launch_k1<R, int16_t, false>(a, n, ntiles, c->stream);
  return mag_out ? launch_k1<R, float, true>(a, n, ntiles, c->stream)
                 : launch_k1<R, float, false>(a, n, ntiles, c->stream);
}

}  // namespace

int afp_launch_stft(afp_ctx* c, const void* pcm, int dtype, double* mag_out, int64_t tile0, int64_t ntiles) {
  if (ntiles <= 0) return AFP_OK;
  const cudaError_t e =
      c->ap.spectrogram_fp32
          ? launch_stft<float>(c, c->d_window_f, c->d_twid_f, pcm, dtype, mag_out, tile0, ntiles)
          : launch_stft<double>(c, c->d_window, c->d_twid, pcm, dtype, mag_out, tile0, ntiles);
  AFP_CUDA(c, e);
  AFP_CUDA(c, cudaGetLastError());
  c->launches++;
  return AFP_OK;
}

int afp_launch_stats(afp_ctx* c, int item0, int nitems) {
  if (nitems <= 0) return AFP_OK;
  const ItemDesc* items = c->d_items.as<ItemDesc>();
  ItemStats* st = c->d_item_stats.as<ItemStats>();
  double* ts = c->d_tile_stats.as<double>();
  afp_stats_kernel<<<(nitems + 7) / 8, 256, 0, c->stream>>>(items, item0, nitems, ts, st, 0);
  AFP_CUDA(c, cudaGetLastError());
  if (c->ap.spectrogram_fp32)
    afp_floorsum_kernel<float><<<dim3((unsigned)nitems, FS_SPLIT), 256, 0, c->stream>>>(
        items, item0, st, c->d_logs.as<float>(), c->d_nyq.as<double>(), ts);
  else
    afp_floorsum_kernel<double><<<dim3((unsigned)nitems, FS_SPLIT), 256, 0, c->stream>>>(
        items, item0, st, c->d_logs.as<double>(), c->d_nyq.as<double>(), ts);
  AFP_CUDA(c, cudaGetLastError());
  afp_stats_kernel<<<(nitems + 7) / 8, 256, 0, c->stream>>>(items, item0, nitems, ts, st, 1);
  AFP_CUDA(c, cudaGetLastError());
  c->launches += 3;
  return AFP_OK;
}

int afp_launch_sgram(afp_ctx* c, double* sgram_out) {
  if (c->nitems == 0 || c->total_frames == 0) return AFP_OK;
  if (c->ap.spectrogram_fp32)
    afp_sgram_kernel<float><<<c->nitems, AFP_NBINS, 0, c->stream>>>(
        c->d_items.as<ItemDesc>(), c->d_item_stats.as<ItemStats>(), c->d_logs.as<float>(), c->ap.hpf_pole, sgram_out);
  else
    afp_sgram_kernel<double><<<c->nitems, AFP_NBINS, 0, c->stream>>>(
        c->d_items.as<ItemDesc>(), c->d_item_stats.as<ItemStats>(), c->d_logs.as<double>(), c->ap.hpf_pole, sgram_out);
  AFP_CUDA(c, cudaGetLastError());
  c->launches++;
  return AFP_OK;
}
