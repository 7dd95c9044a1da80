// PNG decoding shared by the CUDA kernels (png_kernels.cu) and the CPU test harness (tests/cpp/png_harness.cpp, g++).
//
// Semantics are those of cv::imread as the reference calls it (pybind11/pyxivo.cpp:81-85, src/app/vio.cpp:72): colour types 0, 2, 4, 6 at
// 8 or 16 bits, not interlaced; 3-channel output is BGR (grey replicated, RGB swapped, alpha stripped, 16-bit samples keep their high
// byte), 1-channel output (grey and grey + alpha only) is the grey sample.  Ancillary chunks are skipped.  The zlib header and Adler-32 are
// checked and the inflated length must be exactly rows x (1 + cols x bpp); chunk CRCs are NOT checked (libpng does): Adler-32 covers the
// image data and a CRC pass would cost host CPU per frame.
//
// The container walk (parse) is host code.  inflate() is written once for a group of W::n lanes that run the same bit reader and
// Huffman decoder in lock step (every lane decodes every symbol: same loads, same branches, shared-memory tables written with identical
// values) and split only the output: literals are stored by lane 0, match copies and stored blocks are spread across the lanes, Adler-32
// is summed per lane and reduced.  W = SerialLanes (n = 1) is the plain sequential decoder the CPU harness runs; the kernel uses a warp.
// Every read of compressed input and every write of output is bounds-checked; corrupt input returns a status, never an access outside
// [in, in + n) or [out, out + cap).
#pragma once
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define XB_PNG_HD __host__ __device__ __forceinline__
#else
#define XB_PNG_HD inline
#endif

namespace xb {
namespace png {

// decoder status (0 = ok); png_status_text() names them
enum : int {
  kOk = 0,
  kTruncated,       // compressed data ended early
  kZlibHeader,      // CM != 8, CINFO > 7, FCHECK, or a preset dictionary
  kBlockType,       // reserved block type 3
  kStoredLen,       // stored block LEN != ~NLEN
  kHlit,            // HLIT > 286 literal/length codes
  kHdist,           // HDIST > 30 distance codes
  kOversubscribed,  // over-subscribed code-length set
  kIncomplete,      // incomplete code-length set
  kRepeat,          // code-length repeat with no previous length or past the end
  kNoEndOfBlock,    // literal/length code without a code for end-of-block
  kSymbol,          // invalid literal/length or distance symbol
  kDistance,        // distance before the start of the output
  kTooLong,         // more decompressed bytes than rows x (1 + cols x bpp)
  kTooShort,        // fewer decompressed bytes than rows x (1 + cols x bpp)
  kAdler,           // Adler-32 mismatch
  kFilter,          // row filter type > 4
  kNumStatus
};

inline const char* status_text(int s) {
  switch (s) {
    case kOk: return "ok";
    case kTruncated: return "truncated deflate stream";
    case kZlibHeader: return "bad zlib header";
    case kBlockType: return "invalid deflate block type 3";
    case kStoredLen: return "stored block length does not match its complement";
    case kHlit: return "too many literal/length codes (HLIT > 286)";
    case kHdist: return "too many distance codes (HDIST > 30)";
    case kOversubscribed: return "over-subscribed Huffman code lengths";
    case kIncomplete: return "incomplete Huffman code lengths";
    case kRepeat: return "invalid code-length repeat";
    case kNoEndOfBlock: return "no code for end-of-block";
    case kSymbol: return "invalid literal/length or distance code";
    case kDistance: return "distance too far back";
    case kTooLong: return "too much image data (decompressed length exceeds rows x (1 + cols x bpp))";
    case kTooShort: return "too little image data (decompressed length below rows x (1 + cols x bpp))";
    case kAdler: return "Adler-32 mismatch";
    case kFilter: return "invalid row filter type";
    default: return "unknown error";
  }
}

// ------------------------------------------------------------------------------------------------ container (host)
constexpr int kMaxSide = 16384;                   // larger frames are refused
constexpr unsigned long long kMaxRaw = 1ull << 30;  // rows x (1 + cols x bpp)

struct Info {
  int rows = 0, cols = 0, color_type = 0, bit_depth = 0;
  int channels = 0;  // samples per pixel: 1, 2, 3, 4
  int bpp = 0;       // bytes per pixel = channels x bit_depth / 8
  size_t idat_bytes = 0;
  int n_idat = 0;
  unsigned long long raw_bytes() const { return (unsigned long long)rows * (1 + (unsigned long long)cols * bpp); }
};

inline uint32_t be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

// Walks the chunks of a PNG file of n bytes, validates the container and calls idat(offset, length) for every IDAT payload in order.
// Returns 0, or -1 with *why naming the refusal.
template <class F>
inline int parse(const uint8_t* p, size_t n, Info& I, const char** why, F&& idat) {
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
  I = Info();
  auto fail = [&](const char* w) { *why = w; return -1; };
  if (!p || n < 8) return fail("not a PNG file (shorter than the signature)");
  for (int i = 0; i < 8; ++i)
    if (p[i] != sig[i]) return fail("not a PNG file (bad signature)");
  size_t pos = 8;
  bool seen_ihdr = false, in_idat_run = false, idat_done = false;
  for (;;) {
    if (n - pos < 12) return pos == n ? fail("missing IEND chunk") : fail("chunk runs past the end of the data");
    const uint32_t len = be32(p + pos);
    const uint8_t* ty = p + pos + 4;
    if (len > 0x7fffffffu || len > n - pos - 12) return fail("chunk runs past the end of the data");
    const uint8_t* d = p + pos + 8;
    const bool is_ihdr = !__builtin_memcmp(ty, "IHDR", 4), is_idat = !__builtin_memcmp(ty, "IDAT", 4), is_iend = !__builtin_memcmp(ty, "IEND", 4);
    if (!seen_ihdr) {
      if (!is_ihdr || len != 13) return fail("IHDR missing or not the first chunk");
      seen_ihdr = true;
      const uint32_t w = be32(d), h = be32(d + 4);
      const int bd = d[8], ct = d[9];
      if (w == 0 || h == 0) return fail("zero width or height");
      if (w > (uint32_t)kMaxSide || h > (uint32_t)kMaxSide) return fail("image too large (at most 16384 pixels on a side)");
      if (ct == 3) return fail("palette images are not supported");
      if (ct != 0 && ct != 2 && ct != 4 && ct != 6) return fail("invalid colour type");
      if (bd == 1 || bd == 2 || bd == 4) return fail("bit depths below 8 are not supported");
      if (bd != 8 && bd != 16) return fail("invalid bit depth");
      if (d[10] != 0) return fail("unknown compression method");
      if (d[11] != 0) return fail("unknown filter method");
      if (d[12] == 1) return fail("interlaced (Adam7) images are not supported");
      if (d[12] != 0) return fail("unknown interlace method");
      I.cols = (int)w;
      I.rows = (int)h;
      I.bit_depth = bd;
      I.color_type = ct;
      I.channels = ct == 0 ? 1 : ct == 2 ? 3 : ct == 4 ? 2 : 4;
      I.bpp = I.channels * bd / 8;
      if (I.raw_bytes() > kMaxRaw) return fail("image too large (more than 2^30 bytes of image data)");
    } else if (is_ihdr) {
      return fail("misplaced IHDR chunk");
    } else if (is_idat) {
      if (idat_done) return fail("IDAT chunks are not consecutive");
      in_idat_run = true;
      idat(pos + 8, (size_t)len);
      I.idat_bytes += len;
      I.n_idat++;
    } else if (is_iend) {
      if (!I.n_idat) return fail("missing IDAT chunk");
      return 0;
    } else {
      if (in_idat_run) idat_done = true;
      if (!(ty[0] & 0x20) && __builtin_memcmp(ty, "PLTE", 4)) return fail("unknown critical chunk");
    }
    pos += 12 + (size_t)len;
  }
}

// ------------------------------------------------------------------------------------------------ inflate (host and device)
struct SerialLanes {
  static constexpr int n = 1;
  int lane = 0;
  XB_PNG_HD void sync() const {}
  XB_PNG_HD uint32_t sum(uint32_t v) const { return v; }
};

constexpr int kTableBits = 9;
// canonical Huffman code: counts per length, symbols sorted by code, and a 2^9 lookup table of (symbol << 4 | length) for codes up to
// 9 bits (0 = longer code: walk the counts)
struct Huff {
  uint16_t count[16];
  uint16_t symbol[288];
  uint16_t table[1 << kTableBits];
};

struct Bits {
  const uint8_t* p;
  size_t n, pos;
  uint64_t buf;
  int cnt;
};

XB_PNG_HD void refill(Bits& b) {
  while (b.cnt <= 56 && b.pos < b.n) {
    b.buf |= (uint64_t)b.p[b.pos++] << b.cnt;
    b.cnt += 8;
  }
}
XB_PNG_HD bool need(Bits& b, int k) {
  if (b.cnt < k) refill(b);
  return b.cnt >= k;
}
XB_PNG_HD uint32_t take(Bits& b, int k) {
  const uint32_t v = (uint32_t)(b.buf & ((1ull << k) - 1));
  b.buf >>= k;
  b.cnt -= k;
  return v;
}

// kind 0: code-length code (must be complete); 1: literal/length; 2: distance.  An incomplete literal/length or distance code is accepted
// only when it is a single code of length 1 (or no distance code at all), as zlib does.  The work is split by code length: lane l counts
// the symbols of length l into h.count[l], then assigns their canonical codes in symbol order and fills their table entries (codes are
// prefix-free, so the lanes write disjoint entries).  Every per-length quantity is a scalar: no run-time indexed local arrays.
template <class W>
XB_PNG_HD int build(Huff& h, const uint8_t* len, int n, int kind, const W& w) {
  w.sync();  // len was written by every lane
  for (int l = w.lane; l < 16; l += W::n) {
    int c = 0;
    if (l)
      for (int s = 0; s < n; ++s) c += len[s] == l;
    h.count[l] = (uint16_t)c;
  }
  for (int i = w.lane; i < (1 << kTableBits); i += W::n) h.table[i] = 0;
  w.sync();
  int left = 1, maxl = 0;
  for (int l = 1; l < 16; ++l) {
    left <<= 1;
    left -= h.count[l];
    if (left < 0) return kOversubscribed;
    if (h.count[l]) maxl = l;
  }
  if (left > 0 && (kind == 0 || maxl > 1)) return kIncomplete;
  for (int l = 1 + w.lane; l < 16; l += W::n) {
    int off = 0;
    uint32_t code = 0;
    for (int k = 1; k <= l; ++k) {
      if (k < l) off += h.count[k];
      code = (code + (k > 1 ? h.count[k - 1] : 0)) << 1;
    }
    for (int s = 0; s < n; ++s) {
      if (len[s] != l) continue;
      h.symbol[off++] = (uint16_t)s;
      if (l > kTableBits) continue;
      const uint32_t c = code++;
      uint32_t r = 0;
      for (int k = 0; k < l; ++k) r |= ((c >> k) & 1u) << (l - 1 - k);
      for (uint32_t j = r; j < (1u << kTableBits); j += 1u << l) h.table[j] = (uint16_t)(s << 4 | l);
    }
  }
  w.sync();
  return kOk;
}

// next symbol, or -status
XB_PNG_HD int decode(Bits& b, const Huff& h) {
  if (b.cnt < 15) refill(b);
  const uint32_t e = h.table[b.buf & ((1u << kTableBits) - 1)];
  if (e) {
    const int l = e & 15;
    if (l > b.cnt) return -kTruncated;
    take(b, l);
    return (int)(e >> 4);
  }
  int code = 0, first = 0, index = 0;
  uint64_t bb = b.buf;
  for (int l = 1; l < 16; ++l) {
    code |= (int)(bb & 1);
    bb >>= 1;
    const int c = h.count[l];
    if (code - c < first) {
      if (l > b.cnt) return -kTruncated;
      take(b, l);
      return h.symbol[index + (code - first)];
    }
    index += c;
    first += c;
    first <<= 1;
    code <<= 1;
  }
  return b.cnt >= 15 ? -kSymbol : -kTruncated;
}

// copy len bytes from dist back; the lanes take bytes k = lane, lane + n, ...  For dist >= n every group of n bytes reads only bytes
// written before it; for dist < n byte k repeats out[pos - dist + k % dist].
template <class W>
XB_PNG_HD void copy_match(uint8_t* out, size_t pos, uint32_t len, uint32_t dist, const W& w) {
  w.sync();  // literals of lane 0 and earlier copies are visible to every lane
  if (dist >= (uint32_t)W::n) {
    for (uint32_t base = 0; base < len; base += W::n) {
      const uint32_t k = base + w.lane;
      if (k < len) out[pos + k] = out[pos + k - dist];
      if (base + W::n < len) w.sync();
    }
  } else {
    for (uint32_t k = w.lane; k < len; k += W::n) out[pos + k] = out[pos - dist + k % dist];
  }
}

// zlib stream in[0, n) -> exactly cap bytes at out.  lens: 320 bytes of scratch; lit / dst: tables (shared memory on the device).
template <class W>
XB_PNG_HD int inflate(const uint8_t* in, size_t n, uint8_t* out, size_t cap, Huff& lit, Huff& dst, uint8_t* lens, const W& w) {
  Bits b{in, n, 0, 0, 0};
  if (!need(b, 16)) return kTruncated;
  const uint32_t cmf = take(b, 8), flg = take(b, 8);
  if ((cmf & 15) != 8 || (cmf >> 4) > 7 || ((cmf << 8) | flg) % 31 != 0 || (flg & 32)) return kZlibHeader;
  size_t pos = 0;
  uint32_t last = 0;
  do {
    if (!need(b, 3)) return kTruncated;
    last = take(b, 1);
    const uint32_t type = take(b, 2);
    if (type == 3) return kBlockType;
    if (type == 0) {
      take(b, b.cnt & 7);
      if (!need(b, 32)) return kTruncated;
      uint32_t len = take(b, 16);
      const uint32_t nlen = take(b, 16);
      if (len != (~nlen & 0xffffu)) return kStoredLen;
      if (len > cap - pos) return kTooLong;
      while (len && b.cnt >= 8) {  // whole bytes still in the bit buffer
        const uint8_t v = (uint8_t)take(b, 8);
        if (w.lane == 0) out[pos] = v;
        ++pos;
        --len;
      }
      if (len > b.n - b.pos) return kTruncated;
      for (uint32_t k = w.lane; k < len; k += W::n) out[pos + k] = b.p[b.pos + k];
      pos += len;
      b.pos += len;
      continue;
    }
    int err;
    if (type == 1) {
      for (int s = 0; s < 288; ++s) lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
      for (int s = 0; s < 32; ++s) lens[288 + s] = 5;
      if ((err = build(lit, lens, 288, 1, w)) || (err = build(dst, lens + 288, 32, 2, w))) return err;
    } else {
      if (!need(b, 14)) return kTruncated;
      const int nlen = (int)take(b, 5) + 257, ndist = (int)take(b, 5) + 1, ncode = (int)take(b, 4) + 4;
      if (nlen > 286) return kHlit;
      if (ndist > 30) return kHdist;
      const char* order = "\x10\x11\x12\x00\x08\x07\x09\x06\x0a\x05\x0b\x04\x0c\x03\x0d\x02\x0e\x01\x0f";  // 16 17 18 0 8 7 9 ...
      for (int i = 0; i < 19; ++i) lens[i] = 0;
      for (int i = 0; i < ncode; ++i) {
        if (!need(b, 3)) return kTruncated;
        lens[(uint8_t)order[i]] = (uint8_t)take(b, 3);
      }
      if ((err = build(dst, lens, 19, 0, w))) return err;  // the code-length code lives in dst until the distance code is built
      int idx = 0, prev = -1;
      while (idx < nlen + ndist) {
        const int sym = decode(b, dst);
        if (sym < 0) return -sym;
        if (sym < 16) {
          lens[idx++] = (uint8_t)sym;
          prev = sym;
          continue;
        }
        int rep, v = 0;
        if (sym == 16) {
          if (prev < 0) return kRepeat;
          if (!need(b, 2)) return kTruncated;
          v = prev;
          rep = 3 + (int)take(b, 2);
        } else if (sym == 17) {
          if (!need(b, 3)) return kTruncated;
          rep = 3 + (int)take(b, 3);
        } else {
          if (!need(b, 7)) return kTruncated;
          rep = 11 + (int)take(b, 7);
        }
        if (idx + rep > nlen + ndist) return kRepeat;
        for (int k = 0; k < rep; ++k) lens[idx++] = (uint8_t)v;
        prev = v;
      }
      if (lens[256] == 0) return kNoEndOfBlock;
      if ((err = build(lit, lens, nlen, 1, w)) || (err = build(dst, lens + nlen, ndist, 2, w))) return err;
    }
    for (;;) {
      int sym = decode(b, lit);
      if (sym < 0) return -sym;
      if (sym < 256) {
        if (pos >= cap) return kTooLong;
        if (w.lane == 0) out[pos] = (uint8_t)sym;
        ++pos;
        continue;
      }
      if (sym == 256) break;
      sym -= 257;
      if (sym >= 29) return kSymbol;
      uint32_t len;
      if (sym < 8) len = 3 + sym;
      else if (sym == 28) len = 258;
      else {
        const int e = (sym - 4) >> 2;
        if (!need(b, e)) return kTruncated;
        len = ((4u + (sym & 3)) << e) + 3 + take(b, e);
      }
      const int ds = decode(b, dst);
      if (ds < 0) return -ds;
      if (ds >= 30) return kSymbol;
      uint32_t dist;
      if (ds < 4) dist = 1 + ds;
      else {
        const int e = (ds - 2) >> 1;
        if (!need(b, e)) return kTruncated;
        dist = ((2u + (ds & 1)) << e) + 1 + take(b, e);
      }
      if (dist > pos) return kDistance;
      if (len > cap - pos) return kTooLong;
      copy_match(out, pos, len, dist, w);
      pos += len;
    }
  } while (!last);
  if (pos != cap) return kTooShort;
  // Adler-32 of the output: s1 = 1 + sum d_i, s2 = cap + sum (cap - i) d_i (mod 65521), each lane over a stride of the bytes
  w.sync();
  const uint32_t M = 65521;
  uint64_t s1 = 0, s2 = 0;
  uint32_t k = 0;
  for (size_t i = w.lane; i < cap; i += W::n) {
    const uint32_t d = out[i];
    s1 += d;
    s2 += (uint64_t)(cap - i) * d;
    if (++k == 4096) {
      s1 %= M;
      s2 %= M;
      k = 0;
    }
  }
  const uint32_t a = (uint32_t)((1 + w.sum((uint32_t)(s1 % M))) % M);
  const uint32_t bsum = (uint32_t)((cap % M + w.sum((uint32_t)(s2 % M))) % M);
  take(b, b.cnt & 7);
  if (!need(b, 32)) return kTruncated;
  const uint32_t lo = take(b, 16), hi = take(b, 16);
  const uint32_t want = (lo & 0xff) << 24 | (lo >> 8) << 16 | (hi & 0xff) << 8 | hi >> 8;  // big-endian on the wire
  return want == (bsum << 16 | a) ? kOk : kAdler;
}

// ------------------------------------------------------------------------------------------------ rows
XB_PNG_HD uint32_t predict(int ft, uint32_t a, uint32_t b, uint32_t c) {
  switch (ft) {
    case 1: return a;
    case 2: return b;
    case 3: return (a + b) >> 1;
    case 4: {
      const int p = (int)a + (int)b - (int)c;
      const int pa = p > (int)a ? p - (int)a : (int)a - p, pb = p > (int)b ? p - (int)b : (int)b - p, pc = p > (int)c ? p - (int)c : (int)c - p;
      return (pa <= pb && pa <= pc) ? a : pb <= pc ? b : c;
    }
    default: return 0;
  }
}

// undo filter ft on one row in place (prev = the unfiltered row above, nullptr for the first row)
XB_PNG_HD int unfilter_row(uint8_t* cur, const uint8_t* prev, int ft, size_t rowbytes, int bpp) {
  if (ft > 4) return kFilter;
  for (size_t x = 0; x < rowbytes; ++x) {
    const uint32_t a = x >= (size_t)bpp ? cur[x - bpp] : 0, b = prev ? prev[x] : 0, c = (prev && x >= (size_t)bpp) ? prev[x - bpp] : 0;
    cur[x] = (uint8_t)(cur[x] + predict(ft, a, b, c));
  }
  return kOk;
}

// one pixel of an unfiltered row (channels samples of bps bytes, big-endian) -> oc bytes of the cv::imread result
XB_PNG_HD void convert_px(const uint8_t* px, int channels, int bps, int oc, uint8_t* o) {
  if (oc == 1 || channels <= 2) {
    const uint8_t v = px[0];
    for (int k = 0; k < oc; ++k) o[k] = v;
  } else {
    o[0] = px[2 * bps];
    o[1] = px[bps];
    o[2] = px[0];
  }
}

}  // namespace png
}  // namespace xb
