// FLAC decoding on the device (include/afp.h, "FLAC decoding"): what the reference has `ffmpeg -i F
// -f s16le` do to a FLAC file before its reader sees a sample (audio_read.py:196-203), up to the
// interleaved int16 stream afp_pcm_frontend_batch takes.
//
// afp_flac_locate_batch
//   flac_candidate_kernel  one thread per byte: does a frame header start here?  Sync code, no
//                          reserved value, fields consistent with STREAMINFO and the header's CRC-8.
//                          1 = candidate, 2 = a header with the right CRC-8 but a reserved code.
//   flac_chain_kernel      one thread per file walks its bytes once, keeping the CRC-16 of the open
//                          frame: a frame ends at the next candidate whose number follows on and where
//                          that CRC is 0 (the CRC-16 of a frame, footer included, is 0).  A sync pattern
//                          inside compressed data fails either test, so it never splits a frame.
//                          Writes each frame's byte offset and first sample, and the file's totals.
// afp_flac_decode_batch
//   flac_decode_kernel     one thread per frame: parses the subframes, runs each channel's predictor
//                          into int32 scratch (planar within the frame), then decorrelates the
//                          channels and writes the int16 samples interleaved at the file's offset.
#include <climits>
#include <cstring>

#include "afp_internal.cuh"

namespace {

// One file of a locate / decode call, built on the host.
struct FlacFile {
  int64_t byte_off;     // first byte of the file's frames in the packed bytes
  int64_t nbytes;
  int64_t cand_off;     // first candidate flag of the file (prefix of nbytes)
  int64_t frame_base;   // first entry of the file's frame table (capacity nbytes / 8 + 1)
  int64_t block_base;   // first block of the candidate kernel (prefix of ceil(nbytes / 256))
  int64_t gframe_base;  // decode: first frame of the file in the call's frame space
  int64_t nframes;      // decode: frames of the file (0 when it failed to locate)
  int64_t nsamples;     // decode: samples per channel
  int64_t out_off;      // decode: first byte of the file in the output
  int64_t scratch_off;  // decode: first int32 of the file in the scratch
  int32_t rate, channels, bps, max_bs;
  int32_t status;       // AFP_FLAC_DEPTH when the host refused it
  int32_t pad;
};

struct FlacFrame {
  int64_t byte;         // offset of the frame from the file's first byte
  int64_t sample;       // first sample (per channel) of the frame
};

struct FlacResult {
  int64_t nsamples;
  int32_t nframes;
  int32_t status;
};

struct FrameHdr {
  int64_t number;       // frame number (fixed block size) or first-sample number (variable)
  int32_t blocksize;
  int32_t chmode;       // 0-7: chmode + 1 independent channels; 8 left/side, 9 right/side, 10 mid/side
  int32_t nbytes;       // header bytes, CRC-8 included
  int32_t variable;
};

constexpr int HDR_OK = 0, HDR_NONE = 1, HDR_RESERVED = 2;

// The frame header at p (avail bytes): HDR_OK with its fields when it is a candidate of file f,
// HDR_RESERVED when the header's CRC-8 is right but a field holds a reserved code, else HDR_NONE.
__device__ int parse_header(const uint8_t* p, int64_t avail, const FlacFile& f, FrameHdr& h) {
  if (avail < 6 || p[0] != 0xFF || (p[1] & 0xFE) != 0xF8) return HDR_NONE;
  h.variable = p[1] & 1;
  const int bs_code = p[2] >> 4, sr_code = p[2] & 15, ch_code = p[3] >> 4, ss_code = (p[3] >> 1) & 7;
  bool reserved = bs_code == 0 || sr_code == 15 || ch_code > 10 || ss_code == 3 || (p[3] & 1);
  // the coded number: 1-6 bytes, UTF-8 style, up to 31 bits.  The format allows a 7-byte (36-bit) sample
  // number, but FFmpeg's header reader refuses the 0xFE lead byte, so such a header is not a header here
  int pos = 4;
  const uint32_t b0 = p[pos++];
  int extra;
  uint64_t v;
  if (b0 < 0x80) { extra = 0; v = b0; }
  else if ((b0 & 0xE0) == 0xC0) { extra = 1; v = b0 & 0x1F; }
  else if ((b0 & 0xF0) == 0xE0) { extra = 2; v = b0 & 0x0F; }
  else if ((b0 & 0xF8) == 0xF0) { extra = 3; v = b0 & 0x07; }
  else if ((b0 & 0xFC) == 0xF8) { extra = 4; v = b0 & 0x03; }
  else if ((b0 & 0xFE) == 0xFC) { extra = 5; v = b0 & 0x01; }
  else return HDR_NONE;
  if (avail < pos + extra + 1) return HDR_NONE;
  for (int k = 0; k < extra; ++k) {
    const uint32_t b = p[pos++];
    if ((b & 0xC0) != 0x80) return HDR_NONE;
    v = (v << 6) | (b & 0x3F);
  }
  h.number = (int64_t)v;
  int32_t bs;
  if (bs_code == 1) bs = 192;
  else if (bs_code >= 2 && bs_code <= 5) bs = 576 << (bs_code - 2);
  else if (bs_code == 6) { if (avail < pos + 2) return HDR_NONE; bs = p[pos++] + 1; }
  else if (bs_code == 7) { if (avail < pos + 3) return HDR_NONE; bs = ((p[pos] << 8) | p[pos + 1]) + 1; pos += 2; }
  else bs = 256 << (bs_code - 8);      // 8-15 (0 is reserved and gives no bytes)
  int32_t rate = f.rate;
  switch (sr_code) {
    case 1: rate = 88200; break;
    case 2: rate = 176400; break;
    case 3: rate = 192000; break;
    case 4: rate = 8000; break;
    case 5: rate = 16000; break;
    case 6: rate = 22050; break;
    case 7: rate = 24000; break;
    case 8: rate = 32000; break;
    case 9: rate = 44100; break;
    case 10: rate = 48000; break;
    case 11: rate = 96000; break;
    case 12: if (avail < pos + 2) return HDR_NONE; rate = p[pos++] * 1000; break;
    case 13: if (avail < pos + 3) return HDR_NONE; rate = (p[pos] << 8) | p[pos + 1]; pos += 2; break;
    case 14: if (avail < pos + 3) return HDR_NONE; rate = ((p[pos] << 8) | p[pos + 1]) * 10; pos += 2; break;
    default: break;
  }
  if (avail < pos + 1) return HDR_NONE;
  uint32_t crc = 0;                                  // CRC-8, polynomial x^8 + x^2 + x + 1
  for (int k = 0; k < pos; ++k) {
    crc ^= p[k];
    for (int b = 0; b < 8; ++b) crc = (crc & 0x80) ? ((crc << 1) ^ 0x07) & 0xFF : (crc << 1) & 0xFF;
  }
  if (crc != p[pos]) return HDR_NONE;
  if (reserved || bs > 65535) return HDR_RESERVED;
  int32_t bps = f.bps;
  switch (ss_code) {
    case 1: bps = 8; break;
    case 2: bps = 12; break;
    case 4: bps = 16; break;
    case 5: bps = 20; break;
    case 6: bps = 24; break;
    case 7: bps = 32; break;
    default: break;
  }
  const int32_t nch = ch_code < 8 ? ch_code + 1 : 2;
  if (bps != f.bps || nch != f.channels || rate != f.rate || (f.max_bs >= 16 && bs > f.max_bs)) return HDR_NONE;
  h.blocksize = bs;
  h.chmode = ch_code;
  h.nbytes = pos + 1;
  return HDR_OK;
}

__global__ void __launch_bounds__(256) flac_candidate_kernel(const uint8_t* bytes, const FlacFile* files, int nfiles,
                                                             uint8_t* cand) {
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
  const FlacFile& f = files[s_file];
  const int64_t i = (b - f.block_base) * blockDim.x + threadIdx.x;
  if (i >= f.nbytes) return;
  const uint8_t* p = bytes + f.byte_off;
  uint8_t flag = 0;
  if (p[i] == 0xFF && i + 1 < f.nbytes && (p[i + 1] & 0xFE) == 0xF8) {
    FrameHdr h;
    const int rc = parse_header(p + i, f.nbytes - i, f, h);
    flag = rc == HDR_OK ? 1 : rc == HDR_RESERVED ? 2 : 0;
  }
  cand[f.cand_off + i] = flag;
}

__device__ __forceinline__ uint32_t crc16_table_entry(uint32_t i) {      // polynomial x^16 + x^15 + x^2 + 1
  uint32_t crc = i << 8;
  for (int b = 0; b < 8; ++b) crc = (crc & 0x8000) ? ((crc << 1) ^ 0x8005) & 0xFFFF : (crc << 1) & 0xFFFF;
  return crc;
}

__global__ void __launch_bounds__(64) flac_chain_kernel(const uint8_t* bytes, const uint8_t* cand, const FlacFile* files,
                                                        int nfiles, FlacFrame* frames, FlacResult* res) {
  __shared__ uint16_t t16[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) t16[i] = (uint16_t)crc16_table_entry(i);
  __syncthreads();
  const int fi = blockIdx.x * blockDim.x + threadIdx.x;
  if (fi >= nfiles) return;
  const FlacFile& f = files[fi];
  FlacResult r{0, 0, f.status};
  const int64_t n = f.nbytes;
  if (r.status || n == 0) {
    res[fi] = r;
    return;
  }
  const uint8_t* p = bytes + f.byte_off;
  const uint8_t* cf = cand + f.cand_off;
  FrameHdr h;
  const int rc = parse_header(p, n, f, h);
  if (rc != HDR_OK) {
    r.status = rc == HDR_RESERVED ? AFP_FLAC_RESERVED : AFP_FLAC_CHAIN;
    res[fi] = r;
    return;
  }
  const int variable = h.variable;
  const int64_t cap = n / 8 + 1;
  FlacFrame* tab = frames + f.frame_base;
  int64_t start = 0, sample = 0, expect = h.number + (variable ? h.blocksize : 1);
  int32_t bs = h.blocksize, nfr = 0, status = 0;
  bool seen = false;      // a header that follows on was passed while the CRC was not 0
  bool passed = false;    // a candidate header was passed
  uint32_t crc = t16[p[0]];
  for (int64_t q = 1;; ++q) {
    if (q == n) {
      if (crc != 0) status = seen ? AFP_FLAC_CRC : passed ? AFP_FLAC_CHAIN : AFP_FLAC_TRUNCATED;
      break;
    }
    const uint8_t c = cf[q];
    if (c == 1) {
      FrameHdr g;
      parse_header(p + q, n - q, f, g);
      const bool follows = g.variable == variable && g.number == expect;
      passed = true;
      if (crc == 0) {
        if (!follows || nfr + 1 >= cap) {
          status = AFP_FLAC_CHAIN;
          break;
        }
        tab[nfr++] = FlacFrame{start, sample};
        sample += bs;
        start = q;
        bs = g.blocksize;
        expect = g.number + (variable ? g.blocksize : 1);
        seen = passed = false;
      } else if (follows) {
        seen = true;
      }
    } else if (c == 2 && crc == 0) {
      status = AFP_FLAC_RESERVED;
      break;
    }
    crc = ((crc << 8) ^ t16[((crc >> 8) ^ p[q]) & 0xFF]) & 0xFFFF;
  }
  if (status) {
    r.status = status;
  } else {
    tab[nfr++] = FlacFrame{start, sample};
    r.nsamples = sample + bs;
    r.nframes = nfr;
  }
  res[fi] = r;
}

// MSB-first bit reader over bytes [byte, end) of a frame; reads past `end` give zeros and are caught by
// overrun().
struct BitReader {
  const uint8_t* p;
  int64_t byte, end;
  uint64_t cache;       // left-aligned, nbits valid bits
  int nbits;
  bool bad;

  __device__ __forceinline__ void refill() {
#pragma unroll 1
    while (nbits <= 56) {
      const uint64_t v = byte < end ? p[byte] : 0;
      cache |= v << (56 - nbits);
      nbits += 8;
      ++byte;
    }
  }
  __device__ __forceinline__ bool overrun() const { return bad || byte * 8 - nbits > end * 8; }
  __device__ __forceinline__ uint32_t getu(int n) {      // 0 <= n <= 32
    if (n == 0) return 0;
    refill();
    const uint32_t v = (uint32_t)(cache >> (64 - n));
    cache <<= n;
    nbits -= n;
    return v;
  }
  __device__ __forceinline__ int32_t gets(int n) {
    if (n == 0) return 0;
    return (int32_t)(getu(n) << (32 - n)) >> (32 - n);
  }
  __device__ __forceinline__ uint32_t unary() {          // zeros before the next 1
    uint32_t q = 0;
    for (;;) {
      refill();
      if (cache) {
        const int z = __clzll(cache);
        q += z;
        cache <<= z;
        cache <<= 1;
        nbits -= z + 1;
        return q;
      }
      q += nbits;
      nbits = 0;
      if (overrun()) {
        bad = true;
        return 0;
      }
    }
  }
};

// Residual of a FIXED or LPC subframe into s[order .. bs).
__device__ __forceinline__ int read_residual(BitReader& br, int32_t* s, int bs, int order) {
  const int method = br.getu(2);
  if (method > 1) return AFP_FLAC_RESERVED;
  const int po = br.getu(4);
  const int psize = bs >> po;
  if ((psize << po) != bs || order > psize) return AFP_FLAC_CORRUPT;
  const int kbits = method ? 5 : 4, esc = method ? 31 : 15;
  int i = order;
  for (int part = 0; part < (1 << po); ++part) {
    const int k = br.getu(kbits);
    const int end = (part + 1) * psize;
    if (k == esc) {
      const int nb = br.getu(5);
      for (; i < end; ++i) s[i] = br.gets(nb);
    } else {
      // FFmpeg's Rice reader caps the quotient at limit = 2^(32 - k) + 1 (2^31 - 1 for k < 2): a run of
      // limit zeros is refused, a run of limit - 1 reads one bit b and gives u = b + 1, and u = 2^32 - 1
      // (residual -2^31) is refused.  Both refusals drop the frame there, so they make the file unreadable.
      const uint32_t limit = k > 1 ? (INT_MAX >> (k - 1)) + 2u : (uint32_t)INT_MAX;
      for (; i < end; ++i) {
        const uint32_t q = br.unary();
        if (br.bad || q >= limit) return AFP_FLAC_CORRUPT;
        const uint32_t u = q == limit - 1 ? br.getu(1) + 1 : (q << k) | br.getu(k);
        if (u == 0xFFFFFFFFu) return AFP_FLAC_CORRUPT;
        s[i] = (int32_t)((u >> 1) ^ (0u - (u & 1)));
      }
    }
    if (br.overrun()) return AFP_FLAC_CORRUPT;
  }
  return AFP_FLAC_OK;
}

// One subframe of sbps bits per sample into s[0 .. bs); coef is this thread's 32-entry LPC scratch.
__device__ __forceinline__ int decode_subframe(BitReader& br, int32_t* s, int bs, int sbps, int32_t* coef) {
  if (br.getu(1)) return AFP_FLAC_RESERVED;              // the zero padding bit
  const int type = br.getu(6);
  int wasted = 0;
  if (br.getu(1)) {
    wasted = (int)br.unary() + 1;
    if (br.bad || wasted >= sbps) return AFP_FLAC_CORRUPT;
  }
  sbps -= wasted;
  if (type == 0) {
    const int32_t v = br.gets(sbps);
    for (int i = 0; i < bs; ++i) s[i] = v;
  } else if (type == 1) {
    for (int i = 0; i < bs; ++i) s[i] = br.gets(sbps);
  } else if (type >= 8 && type <= 12) {
    const int order = type - 8;
    if (order > bs) return AFP_FLAC_CORRUPT;
    for (int i = 0; i < order; ++i) s[i] = br.gets(sbps);
    const int rc = read_residual(br, s, bs, order);
    if (rc) return rc;
    int64_t a1 = order > 0 ? s[order - 1] : 0, a2 = order > 1 ? s[order - 2] : 0;
    int64_t a3 = order > 2 ? s[order - 3] : 0, a4 = order > 3 ? s[order - 4] : 0;
    for (int i = order; i < bs; ++i) {
      int64_t pr;
      switch (order) {
        case 0: pr = 0; break;
        case 1: pr = a1; break;
        case 2: pr = 2 * a1 - a2; break;
        case 3: pr = 3 * a1 - 3 * a2 + a3; break;
        default: pr = 4 * a1 - 6 * a2 + 4 * a3 - a4; break;
      }
      const int32_t v = (int32_t)(s[i] + pr);
      s[i] = v;
      a4 = a3;
      a3 = a2;
      a2 = a1;
      a1 = v;
    }
  } else if (type >= 32) {
    const int order = (type & 31) + 1;
    if (order > bs) return AFP_FLAC_CORRUPT;
    for (int i = 0; i < order; ++i) s[i] = br.gets(sbps);
    const int prec = br.getu(4);
    if (prec == 15) return AFP_FLAC_RESERVED;
    const int shift = br.gets(5);
    if (shift < 0) return AFP_FLAC_CORRUPT;
    for (int j = 0; j < order; ++j) coef[j] = br.gets(prec + 1);
    const int rc = read_residual(br, s, bs, order);
    if (rc) return rc;
    for (int i = order; i < bs; ++i) {
      int64_t sum = 0;
      for (int j = 0; j < order; ++j) sum += (int64_t)coef[j] * s[i - 1 - j];
      s[i] = (int32_t)(s[i] + (sum >> shift));
    }
  } else {
    return AFP_FLAC_RESERVED;
  }
  if (br.overrun()) return AFP_FLAC_CORRUPT;
  if (wasted)
    for (int i = 0; i < bs; ++i) s[i] = (int32_t)((uint32_t)s[i] << wasted);
  return AFP_FLAC_OK;
}

constexpr int DECODE_THREADS = 128;

__global__ void __launch_bounds__(DECODE_THREADS) flac_decode_kernel(const uint8_t* bytes, const FlacFile* files,
                                                                     int nfiles, const FlacFrame* frames,
                                                                     int64_t total_frames, int32_t* scratch,
                                                                     uint8_t* out, int full_depth, int32_t* status) {
  __shared__ int32_t s_coef[DECODE_THREADS][33];
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total_frames) return;
  int lo = 0, hi = nfiles - 1;                 // the last file whose first frame is <= g
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (files[mid].gframe_base <= g) lo = mid; else hi = mid - 1;
  }
  const FlacFile& f = files[lo];
  const int64_t k = g - f.gframe_base;
  const FlacFrame fr = frames[f.frame_base + k];
  const int64_t fend = k + 1 < f.nframes ? frames[f.frame_base + k + 1].byte : f.nbytes;
  const uint8_t* p = bytes + f.byte_off + fr.byte;
  FrameHdr h;
  int rc = parse_header(p, fend - fr.byte, f, h);
  const int bs = h.blocksize, nch = f.channels;
  if (rc != HDR_OK || fr.sample + bs > f.nsamples) {
    atomicMin(status + lo, AFP_FLAC_CORRUPT);
    return;
  }
  BitReader br{p, h.nbytes, fend - fr.byte - 2, 0, 0, false};       // the body, without the CRC-16
  int32_t* s = scratch + f.scratch_off + fr.sample * nch;           // channel c at s[c * bs + i]
#pragma unroll 1
  for (int c = 0; c < nch && !rc; ++c) {
    const bool side = (h.chmode == 8 && c == 1) || (h.chmode == 9 && c == 0) || (h.chmode == 10 && c == 1);
    rc = decode_subframe(br, s + (int64_t)c * bs, bs, f.bps + (side ? 1 : 0), s_coef[threadIdx.x]);
  }
  if (rc) {
    atomicMin(status + lo, rc);
    return;
  }
  const int bps = f.bps;
  const bool s32 = full_depth && bps > 16;          // x << (32 - bps), as FFmpeg's decoder gives it
  uint8_t* o = out + f.out_off + fr.sample * nch * (s32 ? 4 : 2);
  for (int i = 0; i < bs; ++i) {
    for (int c = 0; c < nch; ++c) {
      int32_t v = s[(int64_t)c * bs + i];
      if (h.chmode >= 8) {
        const int32_t a = s[i], b = s[bs + i];
        if (h.chmode == 8) v = c == 0 ? a : a - b;                       // left, side
        else if (h.chmode == 9) v = c == 0 ? a + b : b;                  // side, right
        else {                                                           // mid, side
          const int32_t mid = (int32_t)(((uint32_t)a << 1) | (uint32_t)(b & 1));
          v = c == 0 ? (mid + b) >> 1 : (mid - b) >> 1;
        }
      }
      if (s32)
        reinterpret_cast<int32_t*>(o)[(int64_t)i * nch + c] = (int32_t)((uint32_t)v << (32 - bps));
      else
        reinterpret_cast<int16_t*>(o)[(int64_t)i * nch + c] =
            (int16_t)(bps <= 16 ? (int32_t)((uint32_t)v << (16 - bps)) : v >> (bps - 16));
    }
  }
}

const char* flac_reason(int s) {
  switch (s) {
    case AFP_FLAC_DEPTH: return "bits per sample outside 4-24";
    case AFP_FLAC_CHAIN: return "broken frame chain";
    case AFP_FLAC_CRC: return "frame CRC-16 mismatch";
    case AFP_FLAC_RESERVED: return "reserved code";
    case AFP_FLAC_TRUNCATED: return "truncated last frame";
    default: return "subframe data does not fit its frame";
  }
}

// AFP_OK, or the code and message of the lowest failing file.
int flac_first_failure(afp_ctx* c, const std::vector<int32_t>& st) {
  for (size_t f = 0; f < st.size(); ++f)
    if (st[f])
      AFP_FAIL(c, st[f] == AFP_FLAC_DEPTH ? AFP_ERR_UNSUPPORTED : AFP_ERR_INVALID,
               "FLAC file " + std::to_string(f) + ": " + flac_reason(st[f]));
  return AFP_OK;
}

}  // namespace

extern "C" int afp_flac_locate_batch(afp_ctx* c, const uint8_t* bytes, int bytes_on_host, int64_t nbytes_total,
                                     int32_t nfiles, const afp_flac_stream* files, int64_t* nsamples,
                                     int32_t* file_status) {
  if (!c) return AFP_ERR_INVALID;
  c->fl.valid = false;
  if (nfiles < 0 || nbytes_total < 0) AFP_FAIL(c, AFP_ERR_INVALID, "negative count");
  if (nfiles > 0 && !files) AFP_FAIL(c, AFP_ERR_INVALID, "null file table");
  std::vector<FlacFile> d((size_t)nfiles);
  int64_t cand = 0, frames = 0, blocks = 0;
  for (int f = 0; f < nfiles; ++f) {
    const afp_flac_stream& s = files[f];
    const std::string who = "file " + std::to_string(f);
    if (s.nbytes < 0 || s.byte_offset < 0 || s.byte_offset > nbytes_total || s.nbytes > nbytes_total - s.byte_offset)
      AFP_FAIL(c, AFP_ERR_INVALID, who + ": byte range outside the buffer");
    if (s.channels < 1 || s.channels > 8 || s.sample_rate < 1)
      AFP_FAIL(c, AFP_ERR_INVALID, who + ": STREAMINFO needs 1-8 channels and a positive rate");
    FlacFile& x = d[(size_t)f];
    memset(&x, 0, sizeof x);
    x.byte_off = s.byte_offset;
    x.nbytes = s.nbytes;
    x.rate = s.sample_rate;
    x.channels = s.channels;
    x.bps = s.bits_per_sample;
    x.max_bs = s.max_blocksize;
    x.status = (s.bits_per_sample < 4 || s.bits_per_sample > 24) ? AFP_FLAC_DEPTH : AFP_FLAC_OK;
    x.cand_off = cand;
    x.frame_base = frames;
    x.block_base = blocks;
    cand += x.nbytes;
    frames += x.nbytes / 8 + 1;
    blocks += x.status ? 0 : (x.nbytes + 255) / 256;
  }
  if (blocks > INT32_MAX) AFP_FAIL(c, AFP_ERR_INVALID, "batch too large for one launch");
  if (cand > 0 && !bytes) AFP_FAIL(c, AFP_ERR_INVALID, "null bytes");
  std::vector<FlacResult> r((size_t)nfiles);
  if (nfiles > 0) {
    AFP_CUDA(c, cudaSetDevice(c->device));
    const uint8_t* dbytes = nullptr;
    int rc = afp_stage(c, c->d_fl_in, bytes, (size_t)nbytes_total, bytes_on_host, &dbytes);
    if (rc) return rc;
    AFP_CUDA(c, c->d_fl_cand.reserve((size_t)cand + 16));
    AFP_CUDA(c, c->d_fl_frame.reserve(sizeof(FlacFrame) * (size_t)frames));
    AFP_CUDA(c, c->d_fl_file.reserve(sizeof(FlacFile) * (size_t)nfiles));
    AFP_CUDA(c, c->d_fl_res.reserve(sizeof(FlacResult) * (size_t)nfiles));
    AFP_CUDA(c, cudaMemcpyAsync(c->d_fl_file.p, d.data(), sizeof(FlacFile) * (size_t)nfiles, cudaMemcpyHostToDevice,
                                c->stream));
    if ((rc = afp_launch(c, flac_candidate_kernel, (unsigned)blocks, 256, 0, dbytes, c->d_fl_file.as<FlacFile>(), nfiles,
                         c->d_fl_cand.as<uint8_t>())) ||
        (rc = afp_launch(c, flac_chain_kernel, (unsigned)((nfiles + 63) / 64), 64, 0, dbytes, c->d_fl_cand.as<uint8_t>(),
                         c->d_fl_file.as<FlacFile>(), nfiles, c->d_fl_frame.as<FlacFrame>(),
                         c->d_fl_res.as<FlacResult>())) ||
        (rc = afp_read_back(c, r.data(), c->d_fl_res.as<FlacResult>(), (size_t)nfiles)))
      return rc;
    c->fl.bytes = dbytes;
  }
  c->fl.nfiles = nfiles;
  c->fl.nsamples.assign((size_t)nfiles, 0);
  c->fl.nframes.assign((size_t)nfiles, 0);
  c->fl.status.assign((size_t)nfiles, 0);
  c->fl.desc.resize(sizeof(FlacFile) * (size_t)nfiles);
  for (int f = 0; f < nfiles; ++f) {
    c->fl.nsamples[f] = r[f].nsamples;
    c->fl.nframes[f] = r[f].nframes;
    c->fl.status[f] = r[f].status;
    if (nsamples) nsamples[f] = r[f].nsamples;
    if (file_status) file_status[f] = r[f].status;
  }
  if (nfiles > 0) memcpy(c->fl.desc.data(), d.data(), c->fl.desc.size());
  c->fl.valid = true;
  return flac_first_failure(c, c->fl.status);
}

extern "C" int afp_flac_decode_batch_bytes(afp_ctx* c, uint8_t* out, int64_t out_capacity, const int64_t* out_offsets,
                                           int32_t full_depth, int32_t* file_status) {
  if (!c) return AFP_ERR_INVALID;
  if (!c->fl.valid) AFP_FAIL(c, AFP_ERR_STATE, "no located FLAC batch (afp_flac_locate_batch)");
  const int nfiles = c->fl.nfiles;
  if (nfiles > 0 && !out_offsets) AFP_FAIL(c, AFP_ERR_INVALID, "null out_offsets");
  std::vector<FlacFile> d((size_t)nfiles);
  if (nfiles > 0) memcpy(d.data(), c->fl.desc.data(), c->fl.desc.size());
  int64_t gframes = 0, scratch = 0;
  for (int f = 0; f < nfiles; ++f) {
    FlacFile& x = d[(size_t)f];
    x.nframes = c->fl.status[f] ? 0 : c->fl.nframes[f];
    x.nsamples = c->fl.status[f] ? 0 : c->fl.nsamples[f];
    x.gframe_base = gframes;
    x.scratch_off = scratch;
    x.out_off = out_offsets[f];
    const int64_t len = x.nsamples * x.channels, width = full_depth && x.bps > 16 ? 4 : 2;
    if (len > 0 && (x.out_off < 0 || x.out_off > out_capacity || len > (out_capacity - x.out_off) / width))
      AFP_FAIL(c, AFP_ERR_INVALID, "file " + std::to_string(f) + ": output range outside the buffer");
    if (len > 0 && (reinterpret_cast<uintptr_t>(out) + (uintptr_t)x.out_off) % (uintptr_t)width)
      AFP_FAIL(c, AFP_ERR_INVALID, "file " + std::to_string(f) + ": output not aligned to its sample width");
    gframes += x.nframes;
    scratch += len;
  }
  if (gframes > 0 && !out) AFP_FAIL(c, AFP_ERR_INVALID, "null output");
  if ((gframes + DECODE_THREADS - 1) / DECODE_THREADS > INT32_MAX)
    AFP_FAIL(c, AFP_ERR_INVALID, "batch too large for one launch");
  std::vector<int32_t> st(c->fl.status);
  if (gframes > 0) {
    AFP_CUDA(c, cudaSetDevice(c->device));
    AFP_CUDA(c, c->d_fl_scratch.reserve(sizeof(int32_t) * (size_t)scratch));
    AFP_CUDA(c, c->d_fl_file.reserve(sizeof(FlacFile) * (size_t)nfiles));
    AFP_CUDA(c, c->d_fl_res.reserve(sizeof(int32_t) * (size_t)nfiles));
    AFP_CUDA(c, cudaMemcpyAsync(c->d_fl_file.p, d.data(), sizeof(FlacFile) * (size_t)nfiles, cudaMemcpyHostToDevice,
                                c->stream));
    AFP_CUDA(c, cudaMemsetAsync(c->d_fl_res.p, 0x7F, sizeof(int32_t) * (size_t)nfiles, c->stream));  // "no failure"
    std::vector<int32_t> dst((size_t)nfiles);
    int rc;
    if ((rc = afp_launch(c, flac_decode_kernel, (unsigned)((gframes + DECODE_THREADS - 1) / DECODE_THREADS),
                         DECODE_THREADS, 0, c->fl.bytes, c->d_fl_file.as<FlacFile>(), nfiles,
                         c->d_fl_frame.as<FlacFrame>(), gframes, c->d_fl_scratch.as<int32_t>(), out, full_depth,
                         c->d_fl_res.as<int32_t>())) ||
        (rc = afp_read_back(c, dst.data(), c->d_fl_res.as<int32_t>(), (size_t)nfiles)))   // `d` is pageable, too
      return rc;
    for (int f = 0; f < nfiles; ++f)
      if (!st[f] && dst[f] != 0x7F7F7F7F) st[f] = dst[f];
  }
  if (file_status)
    for (int f = 0; f < nfiles; ++f) file_status[f] = st[f];
  return flac_first_failure(c, st);
}

extern "C" int afp_flac_decode_batch(afp_ctx* c, int16_t* out, int64_t out_capacity, const int64_t* out_offsets,
                                     int32_t* file_status) {
  if (!c) return AFP_ERR_INVALID;
  if (!c->fl.valid) AFP_FAIL(c, AFP_ERR_STATE, "no located FLAC batch (afp_flac_locate_batch)");
  const int nfiles = c->fl.nfiles;
  if (nfiles > 0 && !out_offsets) AFP_FAIL(c, AFP_ERR_INVALID, "null out_offsets");
  if (out_capacity > INT64_MAX / 2) AFP_FAIL(c, AFP_ERR_INVALID, "output capacity too large");
  std::vector<int64_t> boff((size_t)nfiles + 1);
  for (int f = 0; f < nfiles; ++f) boff[f] = out_offsets[f] < 0 ? -1 : out_offsets[f] > INT64_MAX / 2 ? INT64_MAX : 2 * out_offsets[f];
  return afp_flac_decode_batch_bytes(c, reinterpret_cast<uint8_t*>(out), 2 * out_capacity, boff.data(), 0, file_status);
}
