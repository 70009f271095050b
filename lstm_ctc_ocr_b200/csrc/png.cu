// PNG files decoded to 8-bit gray on the device, sm_90a: byte for byte what cv2.imread(path, 0) (rule 0) or Pillow's
// convert("L") (rule 1) give; the rules and the status codes are in include/crnn_ctc.h.
//
// png_decode_kernel: one warp per file, four files per CTA.  The warp runs one control flow: every lane holds the same chunk
// position, bit buffer and Huffman state (the values are read through broadcast loads), and the lanes split the byte work.
//   chunk walk   per chunk: lane k takes the k-th 32nd of the type + data bytes, table CRC-32 from a zero register, and the
//                lane CRCs are combined by multiplying each by x^(8 * bytes after it) mod P (zlib's crc32_combine algebra);
//                IDAT payloads are copied warp-wide into the file's zlib region
//   inflate      zlib header, then stored / fixed / dynamic blocks (canonical Huffman decode, counts and symbols in shared
//                memory, built by lane 0); literals by lane 0, match and stored copies warp-wide in pieces of min(distance,
//                32) bytes; Adler-32 per lane over a 32nd of the output, combined
//   scanlines    per row of each Adam7 pass: None / Up column-parallel, Sub as a warp scan per byte of a pixel, Average and
//                Paeth serial along the row on bpp lanes; then expansion, the gray rule and the scatter into `out`
// Any failure zeroes the file's slot and sets its status; the other files of the call are not affected.
#include "common.cuh"
#include <stdint.h>

namespace {

constexpr int PNG_WARPS = 4;                 // files per CTA
constexpr int PNG_MAX_H = 1024;              // the images feed's tallest line
constexpr int64_t PNG_MAX_W = 1000000;       // libpng's default user limit
constexpr int64_t PNG_MAX_PIXELS = 178956970;  // 2 x Pillow's MAX_IMAGE_PIXELS: beyond it Image.open raises
// Pillow (rule 1) raises on a zTXt, iTXt or iCCP payload that inflates past MAX_TEXT_CHUNK (1 MiB) and on text chunks that hold
// more than MAX_TEXT_MEMORY (64 MiB) in all.  DEFLATE inflates a byte to at most 1032 (a 258-byte match in two 1-bit codes), so a
// compressed payload of at most 1016 bytes stays under the first limit; a larger one is refused, as are files whose text may pass
// the second.
constexpr int64_t PIL_TEXT_CHUNK = 1 << 20;
constexpr int64_t PIL_TEXT_MEMORY = 64 * PIL_TEXT_CHUNK;
constexpr int64_t DEFLATE_MAX_RATIO = 1032;
constexpr uint32_t CRC_POLY = 0xEDB88320u;
constexpr uint32_t ADLER_MOD = 65521u;

__host__ __device__ inline uint32_t be32(const uint8_t* p) {
  return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | (uint32_t)p[3];
}
__host__ __device__ inline int64_t round16(int64_t n) { return (n + 15) & ~(int64_t)15; }
__host__ __device__ inline int png_channels(int ctype) { return ctype == 2 ? 3 : ctype == 4 ? 2 : ctype == 6 ? 4 : 1; }

// Adam7 pass p: (x0, y0, dx, dy); a non-interlaced image is one pass (0, 0, 1, 1)
__host__ __device__ inline void png_pass(int interlace, int p, int& x0, int& y0, int& dx, int& dy) {
  if (!interlace) { x0 = y0 = 0; dx = dy = 1; return; }
  const int X0[7] = {0, 4, 0, 2, 0, 1, 0}, Y0[7] = {0, 0, 4, 0, 2, 0, 1}, DX[7] = {8, 8, 4, 4, 2, 2, 1}, DY[7] = {8, 8, 8, 4, 4, 2, 2};
  x0 = X0[p]; y0 = Y0[p]; dx = DX[p]; dy = DY[p];
}

// The inflated size of an image (its filter bytes and packed rows over the non-empty passes), or -1 for IHDR data that is
// invalid or beyond the decoder's limits.
__host__ __device__ inline int64_t png_raw_len(const uint8_t* ihdr) {
  const uint32_t w = be32(ihdr), h = be32(ihdr + 4);
  const int depth = ihdr[8], ctype = ihdr[9];
  if (w == 0 || h == 0 || h > PNG_MAX_H || w > PNG_MAX_W || (int64_t)w * h > PNG_MAX_PIXELS) return -1;
  bool ok;
  switch (ctype) {
    case 0: ok = depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16; break;
    case 3: ok = depth == 1 || depth == 2 || depth == 4 || depth == 8; break;
    case 2: case 4: case 6: ok = depth == 8 || depth == 16; break;
    default: ok = false;
  }
  if (!ok || ihdr[10] != 0 || ihdr[11] != 0 || ihdr[12] > 1) return -1;
  const int interlace = ihdr[12], bits = png_channels(ctype) * depth;
  int64_t n = 0;
  for (int p = 0; p < (interlace ? 7 : 1); ++p) {
    int x0, y0, dx, dy;
    png_pass(interlace, p, x0, y0, dx, dy);
    const int64_t pw = ((int64_t)w - x0 + dx - 1) / dx, ph = ((int64_t)h - y0 + dy - 1) / dy;
    if (pw > 0 && ph > 0) n += ph * (1 + (pw * bits + 7) / 8);
  }
  return n;
}

// ---- CRC-32 (reflected, polynomial 0xEDB88320) in GF(2): multiply mod P, and x^(2^k) mod P for k = 0 .. 31
__device__ uint32_t crc_multmodp(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = (b & 1) ? (b >> 1) ^ CRC_POLY : b >> 1;
  }
  return p;
}
__device__ uint32_t crc_x8nmodp(int64_t n, const uint32_t* x2n) {   // x^(8 n) mod P
  uint32_t p = 1u << 31;
  int k = 3;
  while (n) {
    if (n & 1) p = crc_multmodp(x2n[k & 31], p);
    n >>= 1;
    ++k;
  }
  return p;
}

// The CRC-32 of n bytes at q, across the warp (every lane returns it).
__device__ uint32_t warp_crc32(const uint8_t* q, int64_t n, const uint32_t* table, const uint32_t* x2n, int lane) {
  const int64_t seg = (n + 31) / 32, b = min(n, seg * lane), e = min(n, b + seg);
  uint32_t r = 0;
  for (int64_t j = b; j < e; ++j) r = table[(r ^ q[j]) & 255u] ^ (r >> 8);
  r = e > b ? crc_multmodp(crc_x8nmodp(n - e, x2n), r) : 0u;
  for (int o = 16; o; o >>= 1) r ^= __shfl_xor_sync(0xffffffffu, r, o);
  return r ^ crc_multmodp(crc_x8nmodp(n, x2n), 0xFFFFFFFFu) ^ 0xFFFFFFFFu;
}

// ---- inflate
struct Huff {
  short count[16];
  short symbol[288];
};
struct WarpSmem {
  Huff lit, dist;
  uint8_t lens[32 + 286 + 30];   // the code length code's, then the literal/length and distance code lengths
};

struct Bits {                 // identical in every lane
  const uint8_t* in;
  int64_t pos, len;           // next byte to load, stream length
  uint64_t buf;
  int cnt;                    // bits in buf; negative once the stream has been read past its end
  __device__ void refill() {
    while (cnt <= 56 && pos < len) {
      buf |= (uint64_t)in[pos++] << cnt;
      cnt += 8;
    }
  }
  __device__ uint32_t get(int n) {   // n <= 32 bits, after refill(); reading past the end leaves cnt < 0
    const uint32_t v = (uint32_t)(buf & ((n == 32) ? 0xFFFFFFFFull : ((1ull << n) - 1)));
    buf >>= n;
    cnt -= n;
    return v;
  }
};

// puff's canonical code: returns 0 for complete, > 0 incomplete, < 0 over-subscribed.  Lane 0 builds it.
__device__ int huff_build(Huff& hf, const uint8_t* lens, int n, int lane) {
  int left = 1;
  if (lane == 0) {
    short offs[16];
    for (int l = 0; l < 16; ++l) hf.count[l] = 0;
    for (int s = 0; s < n; ++s) hf.count[lens[s]]++;
    for (int l = 1; l < 16; ++l) {
      left <<= 1;
      left -= hf.count[l];
      if (left < 0) break;
    }
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + hf.count[l];
    if (left >= 0)
      for (int s = 0; s < n; ++s)
        if (lens[s]) hf.symbol[offs[lens[s]]++] = (short)s;
  }
  __syncwarp();
  return __shfl_sync(0xffffffffu, left, 0);
}
__device__ __forceinline__ int huff_codes(const Huff& hf) {
  int c = 0;
  for (int l = 1; l < 16; ++l) c += hf.count[l];
  return c;
}
// zlib accepts an incomplete literal/length or distance code only when it is a single code of length 1
__device__ __forceinline__ bool huff_ok(int left, const Huff& hf) { return left == 0 || (left > 0 && hf.count[1] == 1 && huff_codes(hf) == 1); }

__device__ __forceinline__ int huff_decode(Bits& br, const Huff& hf) {   // -1: no code
  int code = 0, first = 0, index = 0;
  for (int l = 1; l < 16; ++l) {
    code |= (int)br.get(1);
    const int count = hf.count[l];
    if (code - count < first) return hf.symbol[index + (code - first)];
    index += count;
    first += count;
    first <<= 1;
    code <<= 1;
  }
  return -1;
}

__constant__ short kLenBase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ short kDistBase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
                                    4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t kClenOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// Inflate z[0, zlen) into raw[0, cap); returns a status, *outlen the bytes written.
__device__ int warp_inflate(const uint8_t* z, int64_t zlen, uint8_t* raw, int64_t cap, WarpSmem& sm, int lane, int64_t* outlen) {
  *outlen = 0;
  if (zlen < 2) return CRNN_PNG_BAD_ZLIB;
  const uint32_t cmf = z[0], flg = z[1];
  if ((cmf & 15) != 8 || (cmf >> 4) > 7 || ((cmf << 8) | flg) % 31 != 0 || (flg & 0x20)) return CRNN_PNG_BAD_ZLIB;
  const int64_t window = (int64_t)1 << ((cmf >> 4) + 8);
  Bits br{z, 2, zlen, 0ull, 0};
  int64_t o = 0;
  bool last = false;
  while (!last) {
    br.refill();
    last = br.get(1);
    const uint32_t type = br.get(2);
    if (br.cnt < 0) return CRNN_PNG_BAD_DEFLATE;
    if (type == 0) {                                 // stored: to the byte boundary, LEN, NLEN, LEN bytes
      br.get(br.cnt & 7);
      int64_t p = br.pos - br.cnt / 8;               // the stream position of the next unread byte
      if (p + 4 > zlen) return CRNN_PNG_BAD_DEFLATE;
      const uint32_t n = z[p] | ((uint32_t)z[p + 1] << 8), nn = z[p + 2] | ((uint32_t)z[p + 3] << 8);
      p += 4;
      if (n != (~nn & 0xFFFFu) || p + n > zlen) return CRNN_PNG_BAD_DEFLATE;
      if (o + n > cap) return CRNN_PNG_BAD_SIZE;
      for (uint32_t j = lane; j < n; j += 32) raw[o + j] = z[p + j];
      o += n;
      br.pos = p + n;
      br.buf = 0;
      br.cnt = 0;
      __syncwarp();
      continue;
    }
    if (type == 3) return CRNN_PNG_BAD_DEFLATE;
    if (type == 1) {                                 // fixed codes
      if (lane == 0) {
        for (int s = 0; s < 144; ++s) sm.lens[s] = 8;
        for (int s = 144; s < 256; ++s) sm.lens[s] = 9;
        for (int s = 256; s < 280; ++s) sm.lens[s] = 7;
        for (int s = 280; s < 288; ++s) sm.lens[s] = 8;
        for (int s = 0; s < 30; ++s) sm.lens[288 + s] = 5;
      }
      __syncwarp();
      huff_build(sm.lit, sm.lens, 288, lane);
      huff_build(sm.dist, sm.lens + 288, 30, lane);
    } else {                                         // dynamic codes
      const int nlen = br.get(5) + 257, ndist = br.get(5) + 1, ncode = br.get(4) + 4;
      if (nlen > 286 || ndist > 30) return CRNN_PNG_BAD_DEFLATE;
      uint8_t cl[19];
      for (int s = 0; s < 19; ++s) cl[s] = 0;
      br.refill();
      for (int s = 0; s < ncode; ++s) {
        if ((s & 7) == 0) br.refill();
        cl[kClenOrder[s]] = (uint8_t)br.get(3);
      }
      if (br.cnt < 0) return CRNN_PNG_BAD_DEFLATE;
      if (lane == 0)
        for (int s = 0; s < 19; ++s) sm.lens[s] = cl[s];
      __syncwarp();
      if (huff_build(sm.lit, sm.lens, 19, lane) != 0) return CRNN_PNG_BAD_DEFLATE;   // the code length code must be complete
      uint8_t* L = sm.lens + 32;                     // past the 19 code length code lengths
      int idx = 0;
      while (idx < nlen + ndist) {
        br.refill();
        int sym = huff_decode(br, sm.lit);
        if (sym < 0 || br.cnt < 0) return CRNN_PNG_BAD_DEFLATE;
        if (sym < 16) {
          if (lane == 0) L[idx] = (uint8_t)sym;
          ++idx;
        } else {
          int v = 0, rep;
          if (sym == 16) {
            if (idx == 0) return CRNN_PNG_BAD_DEFLATE;
            __syncwarp();
            v = L[idx - 1];
            rep = 3 + br.get(2);
          } else if (sym == 17) {
            rep = 3 + br.get(3);
          } else {
            rep = 11 + br.get(7);
          }
          if (br.cnt < 0 || idx + rep > nlen + ndist) return CRNN_PNG_BAD_DEFLATE;
          if (lane == 0)
            for (int r = 0; r < rep; ++r) L[idx + r] = (uint8_t)v;
          idx += rep;
        }
      }
      __syncwarp();
      if (L[256] == 0) return CRNN_PNG_BAD_DEFLATE;   // no end-of-block code
      if (!huff_ok(huff_build(sm.lit, L, nlen, lane), sm.lit)) return CRNN_PNG_BAD_DEFLATE;
      const int dl = huff_build(sm.dist, L + nlen, ndist, lane);
      if (!(huff_ok(dl, sm.dist) || huff_codes(sm.dist) == 0)) return CRNN_PNG_BAD_DEFLATE;
    }
    for (;;) {                                       // the block's symbols
      br.refill();
      const int sym = huff_decode(br, sm.lit);
      if (sym < 0 || br.cnt < 0) return CRNN_PNG_BAD_DEFLATE;
      if (sym < 256) {
        if (o >= cap) return CRNN_PNG_BAD_SIZE;
        if (lane == 0) raw[o] = (uint8_t)sym;
        ++o;
        continue;
      }
      if (sym == 256) break;
      const int ls = sym - 257;
      if (ls >= 29) return CRNN_PNG_BAD_DEFLATE;
      const int len = kLenBase[ls] + (int)br.get(kLenExtra[ls]);
      const int ds = huff_decode(br, sm.dist);
      if (ds < 0 || ds >= 30 || br.cnt < 0) return CRNN_PNG_BAD_DEFLATE;
      const int64_t dist = kDistBase[ds] + (int64_t)br.get(kDistExtra[ds]);
      if (br.cnt < 0 || dist > o || dist > window) return CRNN_PNG_BAD_DEFLATE;
      if (o + len > cap) return CRNN_PNG_BAD_SIZE;
      __syncwarp();                                  // the literals lane 0 wrote are visible to the copy
      const int piece = dist < 32 ? (int)dist : 32;
      for (int c = 0; c < len; c += piece) {
        const int n = min(piece, len - c);
        if (lane < n) raw[o + c + lane] = raw[o + c + lane - dist];
        __syncwarp();
      }
      o += len;
    }
  }
  __syncwarp();
  br.get(br.cnt & 7);                                // the Adler-32 starts on a byte boundary
  const int64_t p = br.pos - br.cnt / 8;
  if (br.cnt < 0 || p + 4 != zlen) return CRNN_PNG_BAD_ZLIB;   // a short trailer, or bytes after it
  *outlen = o;
  // Adler-32: lane k sums a 32nd of the output; A = 1 + sum s1_k, B = o + sum (s2_k + s1_k * (bytes after segment k))
  const int64_t seg = (o + 31) / 32, b = min(o, seg * lane), e = min(o, b + seg);
  uint64_t s1 = 0, s2 = 0;
  for (int64_t j = b; j < e; ++j) {
    s1 += raw[j];
    s2 += s1;
    if (((j - b) & 4095) == 4095) { s1 %= ADLER_MOD; s2 %= ADLER_MOD; }
  }
  s1 %= ADLER_MOD;
  s2 = (s2 + s1 * ((uint64_t)(o - e) % ADLER_MOD)) % ADLER_MOD;
  for (int off = 16; off; off >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, off);
    s2 += __shfl_xor_sync(0xffffffffu, s2, off);
  }
  const uint32_t A = (uint32_t)((1 + s1) % ADLER_MOD), B = (uint32_t)(((uint64_t)o % ADLER_MOD + s2) % ADLER_MOD);
  if (((B << 16) | A) != be32(z + zlen - 4)) return CRNN_PNG_BAD_ZLIB;
  if (o != cap) return CRNN_PNG_BAD_SIZE;
  return CRNN_PNG_OK;
}

// ---- scanlines: unfilter in place, then gray into `out`
__device__ __forceinline__ int paeth(int a, int b, int c) {
  const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

__device__ __forceinline__ uint32_t sample(const uint8_t* row, int64_t k, int depth) {   // sample k of a row
  if (depth == 8) return row[k];
  if (depth == 16) return ((uint32_t)row[2 * k] << 8) | row[2 * k + 1];
  const int64_t bit = k * depth;
  return (row[bit >> 3] >> (8 - depth - (int)(bit & 7))) & ((1u << depth) - 1);
}

__device__ __forceinline__ uint32_t gray_rgb(uint32_t r, uint32_t g, uint32_t b, int depth, int rule) {
  if (depth == 16) {
    if (rule == 0) return ((9797u * r + 19234u * g + 3737u * b + 16384u) >> 15) >> 8;
    r >>= 8; g >>= 8; b >>= 8;
  }
  return rule == 0 ? (9797u * r + 19234u * g + 3737u * b) >> 15 : (19595u * r + 38470u * g + 7471u * b + 0x8000u) >> 16;
}

__device__ int warp_scanlines(uint8_t* raw, int h, int w, int depth, int ctype, int interlace, const uint8_t* plte, int npal,
                              int rule, uint8_t* out, int lane) {
  const int ch = png_channels(ctype), bpp = max(1, ch * depth / 8);
  uint8_t* row = raw;
  for (int p = 0; p < (interlace ? 7 : 1); ++p) {
    int x0, y0, dx, dy;
    png_pass(interlace, p, x0, y0, dx, dy);
    const int pw = (w - x0 + dx - 1) / dx, ph = (h - y0 + dy - 1) / dy;
    if (pw <= 0 || ph <= 0) continue;
    const int64_t rb = ((int64_t)pw * ch * depth + 7) / 8;
    const uint8_t* prior = nullptr;
    for (int r = 0; r < ph; ++r, row += rb + 1) {
      const int f = row[0];
      uint8_t* x = row + 1;
      if (f > 4) return CRNN_PNG_BAD_DATA;
      if (f == 2 && prior) {
        for (int64_t j = lane; j < rb; j += 32) x[j] = (uint8_t)(x[j] + prior[j]);
      } else if (f == 1) {                           // per byte of a pixel: an inclusive scan mod 256 over the pixels
        for (int c = 0; c < bpp; ++c) {
          uint32_t carry = 0;
          for (int64_t j0 = 0; j0 * bpp + c < rb; j0 += 32) {
            const int64_t k = (j0 + lane) * bpp + c;
            uint32_t v = k < rb ? x[k] : 0u;
            for (int o = 1; o < 32; o <<= 1) {
              const uint32_t u = __shfl_up_sync(0xffffffffu, v, o);
              if (lane >= o) v += u;
            }
            v += carry;
            if (k < rb) x[k] = (uint8_t)v;
            carry = __shfl_sync(0xffffffffu, v, 31);
          }
        }
      } else if (f == 3 || f == 4) {                 // serial along the row, one lane per byte of a pixel
        if (lane < bpp) {
          int left = 0, ul = 0;
          for (int64_t k = lane; k < rb; k += bpp) {
            const int up = prior ? prior[k] : 0;
            const int pred = f == 3 ? (left + up) >> 1 : paeth(left, up, ul);
            left = (uint8_t)(x[k] + pred);
            x[k] = (uint8_t)left;
            ul = up;
          }
        }
      }
      __syncwarp();
      // expand and convert: lane per pixel of the row
      bool bad = false;
      uint8_t* dst = out + (int64_t)(y0 + r * dy) * w + x0;
      for (int j = lane; j < pw; j += 32) {
        uint32_t g;
        if (ctype == 3) {
          const uint32_t ix = sample(x, j, depth);
          if ((int)ix >= npal) { bad = true; g = 0; }
          else g = gray_rgb(plte[3 * ix], plte[3 * ix + 1], plte[3 * ix + 2], 8, rule);
        } else if (ctype == 0 || ctype == 4) {
          const uint32_t v = sample(x, (int64_t)j * ch, depth);
          g = depth < 8 ? v * 255u / ((1u << depth) - 1) : depth == 8 ? v : (rule == 1 && ctype == 0 ? min(v, 255u) : v >> 8);
        } else {
          g = gray_rgb(sample(x, (int64_t)j * ch, depth), sample(x, (int64_t)j * ch + 1, depth), sample(x, (int64_t)j * ch + 2, depth),
                       depth, rule);
        }
        dst[(int64_t)j * dx] = (uint8_t)g;
      }
      if (__any_sync(0xffffffffu, bad)) return CRNN_PNG_BAD_DATA;
      prior = x;
    }
  }
  return CRNN_PNG_OK;
}

// ---- the chunk walk and the file's status
__host__ __device__ constexpr uint32_t tag(const char (&s)[5]) {
  return ((uint32_t)(uint8_t)s[0] << 24) | ((uint32_t)(uint8_t)s[1] << 16) | ((uint32_t)(uint8_t)s[2] << 8) | (uint32_t)(uint8_t)s[3];
}
__device__ __forceinline__ bool is_type(uint32_t t, const char (&s)[5]) { return t == tag(s); }

__device__ int warp_decode_file(const uint8_t* f, int64_t flen, int h, int w, int rule, uint8_t* out, uint8_t* region,
                                int64_t region_len, const uint32_t* crc_table, const uint32_t* x2n, WarpSmem& sm, int lane) {
  if (flen < 8 + 25 || be32(f) != 0x89504E47u || be32(f + 4) != 0x0D0A1A0Au) return CRNN_PNG_BAD_HEADER;   // the signature
  if (be32(f + 8) != 13 || !is_type(be32(f + 12), "IHDR")) return CRNN_PNG_BAD_HEADER;
  const uint8_t* ih = f + 16;
  const int64_t raw_len = png_raw_len(ih);
  if (raw_len < 0 || (int64_t)be32(ih) != w || (int64_t)be32(ih + 4) != h) return CRNN_PNG_BAD_HEADER;
  const int depth = ih[8], ctype = ih[9], interlace = ih[12];
  const int64_t zcap = round16(flen);
  if (region_len < zcap + raw_len) return CRNN_PNG_WORKSPACE;
  uint8_t* zs = region;
  uint8_t* raw = region + zcap;

  int64_t pos = 8, zlen = 0, plte = -1;
  int npal = 0, idat = 0;                      // idat: 0 none yet, 1 in the IDAT run, 2 after it
  int64_t text_bound = 0;                      // at least the text Pillow holds for the file's text chunks
  bool iend = false, differs = false;
  while (!iend) {
    if (pos + 12 > flen) return CRNN_PNG_BAD_CHUNK;
    const uint32_t len = be32(f + pos), t = be32(f + pos + 4);
    if (len > 0x7FFFFFFFu || pos + 12 + (int64_t)len > flen) return CRNN_PNG_BAD_CHUNK;
    for (int k = 0; k < 4; ++k) {
      const uint8_t c = f[pos + 4 + k];
      if (!((c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z'))) return CRNN_PNG_BAD_CHUNK;
    }
    if (warp_crc32(f + pos + 4, (int64_t)len + 4, crc_table, x2n, lane) != be32(f + pos + 8 + len)) return CRNN_PNG_BAD_CRC;
    const uint8_t* d = f + pos + 8;
    const bool first = pos == 8;
    if (first != is_type(t, "IHDR")) return CRNN_PNG_BAD_CHUNK;
    if (idat == 1 && !is_type(t, "IDAT")) idat = 2;
    if (is_type(t, "IHDR")) {
    } else if (is_type(t, "IDAT")) {
      if (idat == 2 || (ctype == 3 && plte < 0)) return CRNN_PNG_BAD_CHUNK;
      idat = 1;
      for (uint32_t j = lane; j < len; j += 32) zs[zlen + j] = d[j];
      zlen += len;
    } else if (is_type(t, "IEND")) {
      if (len != 0 || idat == 0 || pos + 12 != flen) return CRNN_PNG_BAD_CHUNK;
      iend = true;
    } else if (is_type(t, "PLTE")) {
      if (plte >= 0 || idat || ctype == 0 || ctype == 4 || len == 0 || len % 3 || len / 3 > 256 ||
          (ctype == 3 && (int)(len / 3) > (1 << depth)))
        return CRNN_PNG_BAD_CHUNK;
      plte = pos + 8;
      npal = len / 3;
    } else if (!(f[pos + 4] & 0x20)) {
      return CRNN_PNG_BAD_CHUNK;                 // an unknown critical chunk
    } else {                                     // ancillary: the ones that change neither reader's gray image
      const bool text = is_type(t, "tEXt") || is_type(t, "zTXt") || is_type(t, "iTXt") || is_type(t, "tIME");
      if (idat && !text) return CRNN_PNG_BAD_CHUNK;
      if (is_type(t, "gAMA") || is_type(t, "sRGB") || is_type(t, "iCCP")) {
        if ((is_type(t, "gAMA") && len != 4) || (is_type(t, "sRGB") && len != 1)) return CRNN_PNG_BAD_CHUNK;
        if (rule == 0 && ctype != 0 && ctype != 4) differs = true;   // libpng gamma-corrects RGB and palette -> gray
      } else if (is_type(t, "cHRM")) {
        if (len != 32) return CRNN_PNG_BAD_CHUNK;
      } else if (is_type(t, "pHYs")) {
        if (len != 9) return CRNN_PNG_BAD_CHUNK;
      } else if (is_type(t, "tIME")) {
        if (len != 7) return CRNN_PNG_BAD_CHUNK;
      } else if (is_type(t, "sBIT")) {
        if (len != (uint32_t)(ctype == 3 ? 3 : png_channels(ctype))) return CRNN_PNG_BAD_CHUNK;
      } else if (is_type(t, "tRNS")) {
        if (ctype == 4 || ctype == 6 || (ctype == 0 && len != 2) || (ctype == 2 && len != 6) ||
            (ctype == 3 && (plte < 0 || len == 0 || (int)len > npal)))
          return CRNN_PNG_BAD_CHUNK;
      } else if (is_type(t, "bKGD")) {
        if (len != (uint32_t)(ctype == 3 ? 1 : (ctype == 0 || ctype == 4) ? 2 : 6) || (ctype == 3 && plte < 0)) return CRNN_PNG_BAD_CHUNK;
      } else if (!text && !is_type(t, "iCCP")) {
        differs = true;                          // acTL, eXIf and every chunk whose effect is not pinned
      }
      if (is_type(t, "iCCP") || is_type(t, "zTXt")) {   // keyword of 1 .. 79 bytes, a null, compression method 0
        int64_t k = 0;
        while (k < len && k < 80 && d[k]) ++k;
        if (k == 0 || k >= 80 || k + 2 > len || d[k + 1] != 0) return CRNN_PNG_BAD_CHUNK;
        const int64_t packed = (int64_t)len - (k + 2);
        if (rule == 1 && packed * DEFLATE_MAX_RATIO > PIL_TEXT_CHUNK) differs = true;
        if (is_type(t, "zTXt")) text_bound += min(packed * DEFLATE_MAX_RATIO, PIL_TEXT_CHUNK);
      } else if (is_type(t, "iTXt")) {                  // keyword, a null, the compression flag: compressed unless it is 0
        int64_t k = 0;
        while (k < len && d[k]) ++k;
        if (k + 1 < len && d[k + 1] != 0) {
          if (rule == 1 && (int64_t)len * DEFLATE_MAX_RATIO > PIL_TEXT_CHUNK) differs = true;
          text_bound += min((int64_t)len * DEFLATE_MAX_RATIO, PIL_TEXT_CHUNK);
        } else {
          text_bound += len;
        }
      } else if (is_type(t, "tEXt")) {
        text_bound += len;
      }
    }
    pos += 12 + (int64_t)len;
  }
  if (ctype == 3 && plte < 0) return CRNN_PNG_BAD_CHUNK;
  if (rule == 1 && text_bound > PIL_TEXT_MEMORY) differs = true;
  if (differs) return CRNN_PNG_HOST_DIFFERS;
  __syncwarp();
  int64_t olen;
  const int st = warp_inflate(zs, zlen, raw, raw_len, sm, lane, &olen);
  if (st != CRNN_PNG_OK) return st;
  return warp_scanlines(raw, h, w, depth, ctype, interlace, plte >= 0 ? f + plte : nullptr, npal, rule, out, lane);
}

__global__ void __launch_bounds__(32 * PNG_WARPS)
png_decode_kernel(const uint8_t* __restrict__ files, const int64_t* __restrict__ file_offset, const int64_t* __restrict__ file_len,
                  int N, const int* __restrict__ hs, const int* __restrict__ ws, const int64_t* __restrict__ out_offset, int rule,
                  uint8_t* __restrict__ out, int* __restrict__ status, uint8_t* __restrict__ workspace,
                  const int64_t* __restrict__ ws_offset, size_t bytes) {
  __shared__ uint32_t s_crc[256], s_x2n[32];
  __shared__ WarpSmem s_warp[PNG_WARPS];
  for (int k = threadIdx.x; k < 256; k += blockDim.x) {
    uint32_t c = k;
    for (int b = 0; b < 8; ++b) c = (c & 1) ? (c >> 1) ^ CRC_POLY : c >> 1;
    s_crc[k] = c;
  }
  if (threadIdx.x == 0) {
    uint32_t p = 1u << 30;                      // x^1
    s_x2n[0] = p;
    for (int k = 1; k < 32; ++k) s_x2n[k] = p = crc_multmodp(p, p);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * PNG_WARPS + warp;
  if (i >= N) return;
  const int h = hs[i], w = ws[i];
  uint8_t* dst = out + out_offset[i];
  const int64_t r0 = ws_offset[i], r1 = ws_offset[i + 1];
  int st;
  if (h < 1 || w < 1)
    st = CRNN_PNG_BAD_HEADER;
  else if (r0 < 0 || r1 < r0 || (uint64_t)r1 > bytes)
    st = CRNN_PNG_WORKSPACE;
  else
    st = warp_decode_file(files + file_offset[i], file_len[i], h, w, rule, dst, workspace + r0, r1 - r0, s_crc, s_x2n, s_warp[warp], lane);
  __syncwarp();
  if (st != CRNN_PNG_OK && h >= 1 && w >= 1)
    for (int64_t j = lane; j < (int64_t)h * w; j += 32) dst[j] = 0;
  if (lane == 0) status[i] = st;
}

}  // namespace

extern "C" int crnn_png_plan(const uint8_t* ihdr, const int64_t* file_len, int N, int64_t* ws_offset, size_t* workspace_bytes) {
  if (!ihdr || !file_len || !ws_offset || !workspace_bytes) return crnn_fail(CRNN_INVALID_VALUE, "png_plan: null pointer");
  if (N <= 0) return crnn_fail(CRNN_INVALID_VALUE, "png_plan: N = %d", N);
  int64_t off = 0;
  for (int i = 0; i < N; ++i) {
    ws_offset[i] = off;
    const int64_t raw = png_raw_len(ihdr + 13 * (size_t)i);
    if (raw >= 0 && file_len[i] > 0) off += round16(file_len[i]) + round16(raw);
  }
  ws_offset[N] = off;
  *workspace_bytes = (size_t)off;
  return CRNN_OK;
}

extern "C" int crnn_png_decode_gray_u8(const uint8_t* files, const int64_t* file_offset, const int64_t* file_len, int N, const int* h,
                                       const int* w, const int64_t* out_offset, int rule, uint8_t* out, int* status, void* workspace,
                                       const int64_t* ws_offset, size_t bytes, crnn_stream_t stream) {
  static const char* fn = "png_decode_gray_u8";
  if (!files || !file_offset || !file_len || !h || !w || !out_offset || !out || !status || !workspace || !ws_offset)
    return crnn_fail(CRNN_INVALID_VALUE, "%s: null pointer", fn);
  if (N <= 0) return crnn_fail(CRNN_INVALID_VALUE, "%s: N = %d", fn, N);
  if (rule != 0 && rule != 1) return crnn_fail(CRNN_INVALID_VALUE, "%s: rule = %d (0: OpenCV, 1: Pillow)", fn, rule);
  CRNN_TRY(check_aligned(file_offset, 8, fn, "file_offset"));
  CRNN_TRY(check_aligned(file_len, 8, fn, "file_len"));
  CRNN_TRY(check_aligned(out_offset, 8, fn, "out_offset"));
  CRNN_TRY(check_aligned(ws_offset, 8, fn, "ws_offset"));
  CRNN_TRY(check_aligned(h, 4, fn, "h"));
  CRNN_TRY(check_aligned(w, 4, fn, "w"));
  CRNN_TRY(check_aligned(status, 4, fn, "status"));
  const int blocks = (N + PNG_WARPS - 1) / PNG_WARPS;
  png_decode_kernel<<<blocks, 32 * PNG_WARPS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      files, file_offset, file_len, N, h, w, out_offset, rule, out, status, static_cast<uint8_t*>(workspace), ws_offset, bytes);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
