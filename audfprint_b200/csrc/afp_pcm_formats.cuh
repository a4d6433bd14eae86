// Sample formats of the PCM front-ends (afp.h AFP_PCM_*): one load per format, shared by the default
// front-end (afp_pcm.cu), which takes every sample as an int16, and the ffmpeg front-end (afp_swr.cu),
// which takes it as an int16 or as a float32 as libswresample does.  Samples are read from the packed
// payload bytes as they came from the file: 2 bytes for AFP_PCM_I16, 3 for AFP_PCM_S24 (little-endian,
// any alignment), 4 for AFP_PCM_S32 and AFP_PCM_F32.  Below them, the output layout, checks, upload and
// launch both batched front-ends share.
#pragma once

#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "afp_internal.cuh"

// bytes per sample, and the alignment a file's first byte needs
__host__ __device__ __forceinline__ int pcm_width(int fmt) {
  return fmt == AFP_PCM_I16 ? 2 : fmt == AFP_PCM_S24 ? 3 : 4;
}
__host__ __device__ __forceinline__ int pcm_align(int fmt) { return fmt == AFP_PCM_S24 ? 1 : pcm_width(fmt); }

// Sample i of a 24- or 32-bit integer format as FFmpeg's decoders give it: int32 holding x << (32 - bits).
__device__ __forceinline__ int32_t pcm_s32(const uint8_t* p, int fmt, int64_t i) {
  if (fmt == AFP_PCM_S24) {
    const uint8_t* q = p + 3 * i;
    return (int32_t)(((uint32_t)q[0] << 8) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 24));
  }
  return reinterpret_cast<const int32_t*>(p)[i];
}

// libswresample's packed float -> s16 (x86 cvtps2dq + packssdw): v * 32768 rounded half to even to
// int32, INT32_MIN for NaN, +-Inf or a value outside the int32 range, then saturated to int16.  For every
// finite in-range value this is the clamp of the rounded value.
__device__ __forceinline__ int pcm_s16_rule(float v) {
  const float t = __fmul_rn(v, 32768.0f);
  const int r = (t >= -2147483648.0f && t < 2147483648.0f) ? __float2int_rn(t) : INT32_MIN;
  return min(max(r, -32768), 32767);
}

// libswresample's scalar float -> s16, av_clip_int16((int) lrintf(v * 32768)): rounded to int64 (NaN,
// +-Inf and values outside the int64 range give INT64_MIN), cut to its low 32 bits, clipped.  The library
// takes it for the last n % 16 samples of a buffer of n; it differs from the packed rule only for NaN,
// +-Inf and |v| >= 65536.
__device__ __forceinline__ int pcm_s16_scalar_rule(float v) {
  const float t = __fmul_rn(v, 32768.0f);
  const long long r = (t > -9.2233720368547758e18f && t < 9.2233720368547758e18f) ? __float2ll_rn(t) : 0;
  return min(max((int)(int32_t)(uint32_t)(unsigned long long)r, -32768), 32767);
}

// Sample i as the int16 `ffmpeg -ac 1` gives a mono file of this format at its own rate: x >> 16 of the
// left-justified integer, the packed s16 rule of a float.
__device__ __forceinline__ int pcm_s16(const uint8_t* p, int fmt, int64_t i) {
  if (fmt == AFP_PCM_F32) return pcm_s16_rule(reinterpret_cast<const float*>(p)[i]);
  if (fmt == AFP_PCM_I16) return reinterpret_cast<const int16_t*>(p)[i];
  return pcm_s32(p, fmt, i) >> 16;
}

// Sample i as libswresample's float32: float(x) * 2^-31 of the left-justified integer (x / 32768 exactly
// for int16), a float as it is.
__device__ __forceinline__ float pcm_f32(const uint8_t* p, int fmt, int64_t i) {
  if (fmt == AFP_PCM_F32) return reinterpret_cast<const float*>(p)[i];
  if (fmt == AFP_PCM_I16) return (float)reinterpret_cast<const int16_t*>(p)[i] * (1.0f / 32768.0f);
  return __fmul_rn(__int2float_rn(pcm_s32(p, fmt, i)), 4.656612873077392578125e-10f);
}

// ---- the half both batched front-ends (afp_pcm.cu, afp_swr.cu) share ----------------------------
// One launch covers a list of files: each file's outputs start on a 16-byte boundary of one device buffer
// (the packed float32 layout afp_fingerprint_batch takes), and each block of 256 outputs belongs to one
// file, found from a per-file block prefix.

// What both front-ends know of a file; each kernel's descriptor extends it with its own parameters.
struct PcmFile {
  int64_t in_off;       // first byte of the file in the packed PCM
  int64_t nframes;
  int64_t out_off;      // first output sample (a multiple of 4: 16-byte aligned)
  int64_t nout;
  int64_t block_base;   // first block of the file: the prefix sum of ceil(nout / 256)
  int32_t ch, fmt;
};

// The file of this block: the last one whose block_base <= blockIdx.x (a file without outputs has the same
// base as the next one), found by thread 0 with a binary search over the block prefix.
template <class D>
__device__ __forceinline__ int pcm_block_file(const D* files, int nfiles) {
  __shared__ int s_file;
  const int64_t b = blockIdx.x;
  if (threadIdx.x == 0) {
    int lo = 0, hi = nfiles - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (files[mid].block_base <= b) lo = mid; else hi = mid - 1;
    }
    s_file = lo;
  }
  __syncthreads();
  return s_file;
}

// The host half of a call up to the launch: every file's common fields, checked (a negative length,
// channels < 1, an unknown format, an input range outside the buffer or off its format's alignment), then
// `own(f, tag, x)` checks and fills the front-end's own fields and x.nout; then the output layout, the
// launch-size and capacity checks and the report to out_offsets / out_lengths.  *blocks: the launch's.
template <class D, class Own>
int pcm_batch_layout(afp_ctx* c, const uint8_t* pcm, int on_host, int64_t pcm_bytes, int32_t nfiles,
                     const int64_t* byte_offsets, const int32_t* formats, const int64_t* nframes,
                     const int32_t* channels, Own own, float* out, int64_t out_capacity, int64_t* out_offsets,
                     int64_t* out_lengths, std::vector<D>* d, int64_t* blocks) {
  if (nfiles < 0 || pcm_bytes < 0) AFP_FAIL(c, AFP_ERR_INVALID, "negative count");
  if (nfiles > 0 && (!byte_offsets || !formats || !nframes || !channels))
    AFP_FAIL(c, AFP_ERR_INVALID, "null per-file array");
  d->assign((size_t)nfiles, D{});
  int64_t o = 0, nb = 0;
  int rc;
  for (int f = 0; f < nfiles; ++f) {
    D& x = (*d)[f];
    const std::string tag = "file " + std::to_string(f) + ": ";
    x.in_off = byte_offsets[f];
    x.nframes = nframes[f];
    x.ch = channels[f];
    x.fmt = formats[f];
    if (x.nframes < 0) AFP_FAIL(c, AFP_ERR_INVALID, tag + "negative length");
    if (x.ch < 1) AFP_FAIL(c, AFP_ERR_INVALID, tag + "channels must be >= 1");
    if (x.fmt < AFP_PCM_I16 || x.fmt > AFP_PCM_S32) AFP_FAIL(c, AFP_ERR_INVALID, tag + "unknown sample format");
    if (x.nframes > 0) {
      if (x.in_off < 0 || x.in_off > pcm_bytes || x.nframes > (pcm_bytes - x.in_off) / pcm_width(x.fmt) / x.ch)
        AFP_FAIL(c, AFP_ERR_INVALID, tag + "input range outside the PCM buffer");
      const uintptr_t first = (on_host ? 0 : reinterpret_cast<uintptr_t>(pcm)) + (uintptr_t)x.in_off;
      if (first % (uintptr_t)pcm_align(x.fmt)) AFP_FAIL(c, AFP_ERR_INVALID, tag + "first sample not aligned to its width");
    }
    if ((rc = own(f, tag, x))) return rc;
    x.out_off = o;
    x.block_base = nb;
    o += (x.nout + 3) & ~(int64_t)3;
    nb += (x.nout + 255) / 256;
  }
  if (nb > INT32_MAX) AFP_FAIL(c, AFP_ERR_INVALID, "batch too large for one launch");
  if (out) {
    if (o > out_capacity) AFP_FAIL(c, AFP_ERR_INVALID, "output buffer smaller than the batch's " + std::to_string(o) + " samples");
    if (nb > 0 && !pcm) AFP_FAIL(c, AFP_ERR_INVALID, "null pcm");
  }
  if (out_offsets) {
    for (int f = 0; f < nfiles; ++f) out_offsets[f] = (*d)[f].out_off;
    out_offsets[nfiles] = o;
  }
  if (out_lengths)
    for (int f = 0; f < nfiles; ++f) out_lengths[f] = (*d)[f].nout;
  *blocks = nb;
  return AFP_OK;
}

// The rest of a call with outputs: stage the PCM (host PCM overwrites the staging buffer of the last
// fingerprint batch), upload the descriptors and the coefficient arrays `coef` (pointer, count) one after
// the other in one copy, launch `kernel` over the blocks and synchronise (the upload's source is pageable).
template <class D, class T>
int pcm_batch_launch(afp_ctx* c, void (*kernel)(const uint8_t*, const D*, int, const T*, float*), const uint8_t* pcm,
                     int on_host, int64_t pcm_bytes, const std::vector<D>& d, int64_t blocks,
                     const std::vector<std::pair<const T*, int64_t>>& coef, float* out) {
  AFP_CUDA(c, cudaSetDevice(c->device));
  const uint8_t* dpcm = nullptr;
  int rc;
  if ((rc = afp_stage(c, c->d_pcm_stage, pcm, (size_t)pcm_bytes, on_host, &dpcm))) return rc;
  if (on_host) c->batch_valid = false;
  int64_t ncoef = 0;
  for (const auto& a : coef) ncoef += a.second;
  D* dd = nullptr;
  T* dcoef = nullptr;
  size_t desc_bytes = 0;
  if ((rc = afp_carve(c, c->d_tmp, [&](Carver& k) {
         dd = k.take<D>((int64_t)d.size());
         desc_bytes = k.bytes;
         dcoef = k.take<T>(ncoef);
       })))
    return rc;
  std::vector<char> h(desc_bytes + sizeof(T) * (size_t)ncoef);
  memcpy(h.data(), d.data(), sizeof(D) * d.size());
  size_t pos = desc_bytes;
  for (const auto& a : coef) {
    if (a.second) memcpy(h.data() + pos, a.first, sizeof(T) * (size_t)a.second);
    pos += sizeof(T) * (size_t)a.second;
  }
  AFP_CUDA(c, afp_copy_in(c, reinterpret_cast<char*>(dd), h.data(), h.size(), 1));
  if ((rc = afp_launch(c, kernel, (unsigned)blocks, 256, 0, dpcm, dd, (int)d.size(), dcoef, out))) return rc;
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  return AFP_OK;
}

// The byte form of an int16 call: every file AFP_PCM_I16 at twice its int16 offset.
inline void pcm_i16_layout(int nfiles, const int64_t* offsets, std::vector<int64_t>* boff, std::vector<int32_t>* fmt) {
  boff->assign((size_t)nfiles + 1, 0);
  fmt->assign((size_t)nfiles + 1, AFP_PCM_I16);
  for (int f = 0; f < nfiles; ++f) (*boff)[f] = 2 * offsets[f];
}
