// Sample formats of the PCM front-ends (afp.h AFP_PCM_*): one load per format, shared by the default
// front-end (afp_pcm.cu), which takes every sample as an int16, and the ffmpeg front-end (afp_swr.cu),
// which takes it as an int16 or as a float32 as libswresample does.  Samples are read from the packed
// payload bytes as they came from the file: 2 bytes for AFP_PCM_I16, 3 for AFP_PCM_S24 (little-endian,
// any alignment), 4 for AFP_PCM_S32 and AFP_PCM_F32.
#pragma once

#include <cstdint>
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

// Host check of one file's input range of a byte-form front-end call: a known format, a first byte inside
// the buffer on the format's alignment, and nframes * ch samples inside the buffer.
inline int pcm_check_input(afp_ctx* c, int f, const uint8_t* pcm, int on_host, int64_t pcm_bytes, int64_t off,
                           int fmt, int64_t nframes, int ch) {
  const std::string tag = "file " + std::to_string(f) + ": ";
  if (fmt < AFP_PCM_I16 || fmt > AFP_PCM_S32) AFP_FAIL(c, AFP_ERR_INVALID, tag + "unknown sample format");
  if (nframes == 0) return AFP_OK;
  const int64_t w = pcm_width(fmt);
  if (off < 0 || off > pcm_bytes || nframes > (pcm_bytes - off) / w / ch)
    AFP_FAIL(c, AFP_ERR_INVALID, tag + "input range outside the PCM buffer");
  const uintptr_t first = (on_host ? 0 : reinterpret_cast<uintptr_t>(pcm)) + (uintptr_t)off;
  if (first % (uintptr_t)pcm_align(fmt)) AFP_FAIL(c, AFP_ERR_INVALID, tag + "first sample not aligned to its width");
  return AFP_OK;
}

// The byte form of an int16 call: every file AFP_PCM_I16 at twice its int16 offset.
inline void pcm_i16_layout(int nfiles, const int64_t* offsets, std::vector<int64_t>* boff, std::vector<int32_t>* fmt) {
  boff->assign((size_t)nfiles + 1, 0);
  fmt->assign((size_t)nfiles + 1, AFP_PCM_I16);
  for (int f = 0; f < nfiles; ++f) (*boff)[f] = 2 * offsets[f];
}
