// Baseline and extended-sequential Huffman JPEG files decoded to 8-bit gray on the device, sm_90a: byte for byte what
// cv2.imread(path, 0) (rule 0: libjpeg's JCS_GRAYSCALE output, the Y plane) or Pillow's convert("L") (rule 1: libjpeg-turbo's
// RGB decode, then L24) give; the rules and the status codes are in include/crnn_ctc.h.
//
// jpeg_entropy_kernel  one warp per file, four files per CTA.  Lane 0 walks the markers up to SOS; lanes 0 .. 5 build the scan's
//                      Huffman tables (a 9-bit lookahead table and libjpeg's maxcode / valoffset for longer codes) in shared
//                      memory; the warp zero-fills the file's coefficient region and finds the RSTn markers with a ballot per
//                      32 bytes; then lane k decodes restart segments k, k + 32, ..., every component's symbols, storing the
//                      int16 coefficients of the components the rule needs.
// jpeg_idct_kernel     8 threads per block, libjpeg-turbo's jidctint.c (ISLOW), exact in 32 bits: a column each, then a row
//                      each through shared memory, the range-limit table at the end.  The gray plane goes straight to `out`,
//                      cropped; under rule 1 a colour file's three planes go to the workspace.
// jpeg_finish_kernel   zeroes the slot of every refused file; rule 1 colour: fancy upsampling, jdcolor.c's YCbCr -> RGB, L24.
//
// libjpeg-turbo's SIMD IDCT (what both host readers run on x86-64 and Arm) keeps dequantised coefficients and the first pass's
// outputs in 16 bits and saturates its outputs where jidctint.c wraps them through the range-limit table.  The two agree while
// every dequantised coefficient and first-pass output lies in [-16383, 16383] and every output sum in [-512, 511]; a block
// outside that envelope makes the file CRNN_JPEG_HOST_DIFFERS.  Encoders produce no such blocks from 8-bit pictures.
#include "common.cuh"
#include <stdint.h>

namespace {

constexpr int JPEG_WARPS = 4;          // files per CTA of the entropy kernel
constexpr int JPEG_MAX_H = 1024;       // the images feed's tallest line
constexpr int JPEG_SPLIT = 4;          // CTAs per file in the IDCT and finish kernels
constexpr int64_t JHDR = 512;          // the per-file record at the start of its workspace region (JInfo, rounded up)
constexpr int ENVELOPE = 16383;

__host__ __device__ inline int64_t round16(int64_t n) { return (n + 15) & ~(int64_t)15; }
__host__ __device__ inline int be16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// The frame's geometry from its SOF payload: P, Y (2), X (2), Nf, then Ci, HiVi, Tqi per component.
struct JGeom {
  int h, w, nf, hmax, vmax, mcux, mcuy, colour;   // colour: rule 1 on a 3-component file (three planes, the finish kernel)
  int H[3], V[3], bw[3], bh[3], pw[3], ph[3];
  int64_t coef[3], plane[3], segtab, bytes;       // region offsets and the region's size
};

// Fills g and returns true when the SOF describes a frame the decoder can lay out; the layout depends on the rule.
__host__ __device__ inline bool jpeg_geom(const uint8_t* sof, int rule, JGeom& g) {
  g.h = be16(sof + 1);
  g.w = be16(sof + 3);
  g.nf = sof[5];
  if (sof[0] != 8 || g.h < 1 || g.h > JPEG_MAX_H || g.w < 1 || (g.nf != 1 && g.nf != 3)) return false;
  g.hmax = g.vmax = 1;
  int blocks = 0;
  for (int c = 0; c < g.nf; ++c) {
    g.H[c] = sof[7 + 3 * c] >> 4;
    g.V[c] = sof[7 + 3 * c] & 15;
    if (g.H[c] < 1 || g.H[c] > 4 || g.V[c] < 1 || g.V[c] > 4) return false;
    g.hmax = g.H[c] > g.hmax ? g.H[c] : g.hmax;
    g.vmax = g.V[c] > g.vmax ? g.V[c] : g.vmax;
    blocks += g.H[c] * g.V[c];
  }
  if (g.nf == 3 && blocks > 10) return false;
  g.colour = rule == 1 && g.nf == 3;
  if (g.nf == 1) {          // a non-interleaved scan: one block per MCU whatever the sampling factors say
    g.H[0] = g.V[0] = g.hmax = g.vmax = 1;
  }
  g.mcux = (g.w + 8 * g.hmax - 1) / (8 * g.hmax);
  g.mcuy = (g.h + 8 * g.vmax - 1) / (8 * g.vmax);
  int64_t off = JHDR;
  g.segtab = off;
  off += round16(((int64_t)g.mcux * g.mcuy + 1) * 8);
  const int stored = g.colour ? 3 : 1;
  for (int c = 0; c < g.nf; ++c) {
    g.bw[c] = g.mcux * g.H[c];
    g.bh[c] = g.mcuy * g.V[c];
    g.pw[c] = (int)(((int64_t)g.w * g.H[c] + g.hmax - 1) / g.hmax);
    g.ph[c] = (int)(((int64_t)g.h * g.V[c] + g.vmax - 1) / g.vmax);
    g.coef[c] = g.plane[c] = -1;
  }
  for (int c = 0; c < stored; ++c) {
    g.coef[c] = off;
    off += (int64_t)g.bw[c] * g.bh[c] * 128;
  }
  if (g.colour)
    for (int c = 0; c < 3; ++c) {
      g.plane[c] = off;
      off += (int64_t)g.bw[c] * g.bh[c] * 64;
    }
  g.bytes = off;
  return true;
}

// What the IDCT and finish kernels read of a decoded file, at the start of its region.
struct JInfo {
  int colour, ncomp;                 // ncomp: the stored components
  int bw[3], bh[3], pw[3], ph[3];
  int rh[3], rv[3];                  // hmax / H, vmax / V
  int64_t coef[3], plane[3];
  uint16_t q[3][64];                 // natural order
};
static_assert(sizeof(JInfo) <= JHDR, "JInfo must fit its record");

__constant__ uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ---- Huffman tables: libjpeg's jpeg_make_d_derived_tbl, with a 9-bit lookahead
constexpr int LOOK = 9;
struct HuffD {
  uint16_t look[1 << LOOK];          // (length << 8) | symbol; 0: the code is longer than LOOK bits
  int maxcode[18];                   // -1: no code of that length
  int valoff[17];
  uint8_t val[256];
};
constexpr int MAX_TABLES = 6;        // a 3-component scan names at most 3 DC and 3 AC tables

struct ParseState {                  // what lane 0's marker walk leaves for the warp
  int status, ri, ns, ntab;
  int64_t sos_end;
  int comp[3];                       // frame component of each scan component
  int dct[3], act[3];                // its DC / AC table among the built ones
  int tab_pos[MAX_TABLES], tab_dc[MAX_TABLES];
  int64_t qpos[3];                   // each frame component's DQT values: file position << 1 | 16-bit flag
  uint8_t sof[16];
};

struct WarpSmem {
  HuffD tab[MAX_TABLES];
  ParseState ps;
};

// Builds table t from the DHT bits at `src` (16 counts, then the symbols); returns a status.
__device__ int huff_derive(const uint8_t* src, bool dc, HuffD& t) {
  int code = 0, p = 0;
  for (int k = 0; k < (1 << LOOK); ++k) t.look[k] = 0;
  for (int l = 1; l <= 16; ++l) {
    const int n = src[l - 1];
    if (n) {
      t.valoff[l] = p - code;
      for (int j = 0; j < n; ++j, ++p, ++code) {
        if (code + 1 >= (1 << l)) return CRNN_JPEG_BAD_HUFFMAN;   // over-subscribed, or an all-ones code
        const uint8_t sym = src[16 + p];
        if (dc && sym > 15) return CRNN_JPEG_BAD_HUFFMAN;
        t.val[p] = sym;
        if (l <= LOOK) {
          const int lo = code << (LOOK - l), hi = (code + 1) << (LOOK - l);
          for (int k = lo; k < hi; ++k) t.look[k] = (uint16_t)((l << 8) | sym);
        }
      }
      t.maxcode[l] = code - 1;
    } else {
      t.maxcode[l] = -1;
      t.valoff[l] = 0;
    }
    code <<= 1;
  }
  t.maxcode[17] = 0xFFFFF;
  return CRNN_JPEG_OK;
}

// ---- the entropy-coded data of one restart segment, MSB first, FF00 unstuffed, zeros past the data
struct BitReader {
  const uint8_t* f;
  int64_t pos, end;                  // next byte; end of the data (a marker's fill bytes start there)
  uint64_t buf;
  int cnt, pad;                      // bits in buf (left-aligned); zero bytes appended after the data
  __device__ void refill() {
    while (cnt <= 56) {
      uint32_t b = 0;
      if (pos < end) {
        b = f[pos];
        if (b == 0xFF) {
          if (pos + 1 < end && f[pos + 1] == 0) {
            pos += 2;
          } else {                   // fill bytes before the segment's marker, or FF FF 00: the data ends here
            end = pos;
            continue;
          }
        } else {
          ++pos;
        }
      } else {
        ++pad;
      }
      buf |= (uint64_t)b << (56 - cnt);
      cnt += 8;
    }
  }
  __device__ __forceinline__ uint32_t get(int n) {   // 1 <= n <= 16, after refill()
    const uint32_t v = (uint32_t)(buf >> (64 - n));
    buf <<= n;
    cnt -= n;
    return v;
  }
};

__device__ __forceinline__ int huff_decode(BitReader& br, const HuffD& t) {   // -1: no code
  const uint32_t e = t.look[br.buf >> (64 - LOOK)];
  if (e) {
    br.buf <<= (e >> 8);
    br.cnt -= (e >> 8);
    return e & 255;
  }
  for (int l = LOOK + 1; l <= 16; ++l) {
    const int code = (int)(br.buf >> (64 - l));
    if (code <= t.maxcode[l]) {
      br.buf <<= l;
      br.cnt -= l;
      return t.val[(code + t.valoff[l]) & 255];
    }
  }
  return -1;
}

__device__ __forceinline__ int extend(uint32_t v, int s) { return (int)v < (1 << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v; }

// One block's symbols; coef null: decoded and checked, not stored.
__device__ __forceinline__ int decode_block(BitReader& br, const HuffD& dc, const HuffD& ac, int& pred, int16_t* coef) {
  br.refill();
  int s = huff_decode(br, dc);
  if (s < 0 || s > 11) return CRNN_JPEG_BAD_DATA;
  if (s) pred += extend(br.get(s), s);
  if (coef) coef[0] = (int16_t)pred;
  for (int k = 1; k < 64; ++k) {
    if (br.cnt < 32) br.refill();
    const int rs = huff_decode(br, ac);
    if (rs < 0) return CRNN_JPEG_BAD_DATA;
    const int r = rs >> 4;
    s = rs & 15;
    if (s) {
      k += r;
      if (k > 63 || s > 10) return CRNN_JPEG_BAD_DATA;
      const int v = extend(br.get(s), s);
      if (coef) coef[kNatural[k]] = (int16_t)v;
    } else {
      if (r != 15) break;
      k += 15;
    }
  }
  return CRNN_JPEG_OK;
}

// rule 0: an Exif orientation other than 1 (OpenCV turns the image), or Exif OpenCV might read otherwise.  d: the APP1 payload.
__device__ bool exif_turns(const uint8_t* d, int n) {
  if (n < 6 || d[0] != 'E' || d[1] != 'x' || d[2] != 'i' || d[3] != 'f' || d[4] != 0 || d[5] != 0) return false;
  const uint8_t* t = d + 6;
  const int64_t tl = n - 6;
  if (tl < 8) return true;
  const bool le = t[0] == 'I' && t[1] == 'I';
  if (!le && !(t[0] == 'M' && t[1] == 'M')) return true;
  auto u16 = [&](int64_t o) -> uint32_t { return le ? (t[o] | (t[o + 1] << 8)) : ((t[o] << 8) | t[o + 1]); };
  auto u32 = [&](int64_t o) -> uint32_t { return le ? (u16(o) | (u16(o + 2) << 16)) : ((u16(o) << 16) | u16(o + 2)); };
  const int64_t ifd = u32(4);
  if (ifd + 2 > tl) return true;
  const int64_t cnt = u16(ifd);
  if (ifd + 2 + 12 * cnt > tl) return true;
  for (int64_t j = 0; j < cnt; ++j) {
    const int64_t e = ifd + 2 + 12 * j;
    if (u16(e) == 0x0112) return u16(e + 2) != 3 || u16(e + 8) != 1;
  }
  return false;
}

// Lane 0: SOI to the end of SOS.  Fills ps (tables named by offsets into the file) and returns a status.
__device__ int walk_markers(const uint8_t* f, int64_t flen, int h, int w, int rule, ParseState& ps) {
  if (flen < 4 || f[0] != 0xFF || f[1] != 0xD8) return CRNN_JPEG_BAD_HEADER;
  int64_t dht[8], dqt[4];
  for (int k = 0; k < 8; ++k) dht[k] = -1;
  for (int k = 0; k < 4; ++k) dqt[k] = -1;
  int64_t pos = 2;
  bool sof = false, jfif = false, adobe = false, differs = false;
  int transform = -1;
  const uint8_t* sofp = nullptr;
  ps.ri = 0;
  for (;;) {
    if (pos >= flen || f[pos] != 0xFF) return CRNN_JPEG_BAD_MARKER;
    while (pos < flen && f[pos] == 0xFF) ++pos;
    if (pos >= flen) return CRNN_JPEG_BAD_MARKER;
    const int m = f[pos++];
    if (m == 0x00 || m == 0x01 || (m >= 0xD0 && m <= 0xD9)) return CRNN_JPEG_BAD_MARKER;   // no segment here
    if (pos + 2 > flen) return CRNN_JPEG_BAD_MARKER;
    const int L = be16(f + pos);
    if (L < 2 || pos + L > flen) return CRNN_JPEG_BAD_MARKER;
    const uint8_t* d = f + pos + 2;
    const int n = L - 2;
    if (m == 0xC0 || m == 0xC1) {
      if (sof) return CRNN_JPEG_BAD_MARKER;
      sof = true;
      if (n < 6) return CRNN_JPEG_BAD_HEADER;
      const int nf = d[5];
      if (n != 6 + 3 * nf || nf == 0) return CRNN_JPEG_BAD_HEADER;
      if (d[0] != 8 || be16(d + 1) == 0 || (nf != 1 && nf != 3)) return CRNN_JPEG_UNSUPPORTED;
      for (int c = 0; c < nf; ++c) {
        const int hv = d[7 + 3 * c];
        if ((hv >> 4) < 1 || (hv >> 4) > 4 || (hv & 15) < 1 || (hv & 15) > 4 || d[8 + 3 * c] > 3) return CRNN_JPEG_BAD_HEADER;
        for (int e = 0; e < c; ++e)
          if (d[6 + 3 * e] == d[6 + 3 * c]) return CRNN_JPEG_BAD_HEADER;
      }
      if (be16(d + 1) != h || be16(d + 3) != w) return CRNN_JPEG_BAD_HEADER;
      sofp = d;
    } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xCC) {
      return CRNN_JPEG_UNSUPPORTED;                // progressive, lossless, hierarchical, arithmetic
    } else if (m == 0xCC) {
      return CRNN_JPEG_UNSUPPORTED;                // arithmetic conditioning
    } else if (m == 0xC4) {
      int k = 0;
      while (k < n) {
        if (k + 17 > n) return CRNN_JPEG_BAD_MARKER;
        const int tc = d[k] >> 4, th = d[k] & 15;
        if (tc > 1 || th > 3) return CRNN_JPEG_BAD_HUFFMAN;
        int count = 0;
        for (int l = 1; l <= 16; ++l) count += d[k + l];
        if (count > 256 || k + 17 + count > n) return CRNN_JPEG_BAD_HUFFMAN;
        dht[tc * 4 + th] = pos + 2 + k + 1;
        k += 17 + count;
      }
    } else if (m == 0xDB) {
      int k = 0;
      while (k < n) {
        const int pq = d[k] >> 4, tq = d[k] & 15;
        if (pq > 1 || tq > 3 || k + 1 + 64 * (pq + 1) > n) return CRNN_JPEG_BAD_MARKER;
        dqt[tq] = ((pos + 2 + k + 1) << 1) | pq;
        k += 1 + 64 * (pq + 1);
      }
    } else if (m == 0xDD) {
      if (n != 2) return CRNN_JPEG_BAD_MARKER;
      ps.ri = be16(d);
    } else if (m == 0xDA) {
      if (!sof) return CRNN_JPEG_BAD_HEADER;
      const int nf = sofp[5], ns = n >= 1 ? d[0] : 0;
      if (ns < 1 || ns > nf || n != 1 + 2 * ns + 3) return CRNN_JPEG_BAD_MARKER;
      if (ns < nf) return CRNN_JPEG_UNSUPPORTED;   // the components in several scans
      ps.ns = ns;
      ps.ntab = 0;
      for (int s = 0; s < ns; ++s) {
        int c = -1;
        for (int e = 0; e < nf; ++e)
          if (sofp[6 + 3 * e] == d[1 + 2 * s]) c = e;
        if (c < 0) return CRNN_JPEG_BAD_MARKER;
        for (int e = 0; e < s; ++e)
          if (ps.comp[e] == c) return CRNN_JPEG_BAD_MARKER;
        ps.comp[s] = c;
        const int td = d[2 + 2 * s] >> 4, ta = d[2 + 2 * s] & 15;
        if (td > 3 || ta > 3 || dht[td] < 0 || dht[4 + ta] < 0) return CRNN_JPEG_BAD_MARKER;
        int* slot[2] = {&ps.dct[s], &ps.act[s]};
        const int64_t at[2] = {dht[td], dht[4 + ta]};
        for (int k = 0; k < 2; ++k) {
          int t = -1;
          for (int e = 0; e < ps.ntab; ++e)
            if (ps.tab_pos[e] == at[k] && ps.tab_dc[e] == (k == 0)) t = e;
          if (t < 0) {
            t = ps.ntab++;
            ps.tab_pos[t] = (int)at[k];
            ps.tab_dc[t] = k == 0;
          }
          *slot[k] = t;
        }
      }
      if (d[1 + 2 * ns] != 0 || d[2 + 2 * ns] != 63 || d[3 + 2 * ns] != 0) return CRNN_JPEG_BAD_MARKER;
      for (int c = 0; c < nf; ++c) {
        if (dqt[sofp[8 + 3 * c]] < 0) return CRNN_JPEG_BAD_MARKER;
        ps.qpos[c] = dqt[sofp[8 + 3 * c]];
      }
      if (nf == 3) {                               // libjpeg's colour-space guess: only YCbCr is read
        const bool rgb_ids = sofp[6] == 'R' && sofp[9] == 'G' && sofp[12] == 'B';
        if (!jfif && (adobe ? transform != 1 : rgb_ids)) return CRNN_JPEG_UNSUPPORTED;
      }
      for (int k = 0; k < 16; ++k) ps.sof[k] = k < 6 + 3 * nf ? sofp[k] : 0;
      ps.sos_end = pos + L;
      return rule == 0 && differs ? CRNN_JPEG_HOST_DIFFERS : CRNN_JPEG_OK;
    } else if (m == 0xE0) {
      if (n >= 14 && d[0] == 'J' && d[1] == 'F' && d[2] == 'I' && d[3] == 'F' && d[4] == 0) jfif = true;
    } else if (m == 0xEE) {
      if (n >= 12 && d[0] == 'A' && d[1] == 'd' && d[2] == 'o' && d[3] == 'b' && d[4] == 'e') {
        adobe = true;
        transform = d[11];
      }
    } else if (m == 0xE1) {
      if (exif_turns(d, n)) differs = true;
    } else if ((m >= 0xE2 && m <= 0xEF) || m == 0xFE) {
    } else {
      return CRNN_JPEG_BAD_MARKER;                 // DNL before the scan, JPGn, reserved codes
    }
    pos += L;
  }
}


// After a segment's MCUs: the padding bits of its last byte, then fill bytes up to the marker, and nothing else.
__device__ __forceinline__ int segment_tail(const uint8_t* f, const BitReader& br, int64_t seg_end) {
  if (br.cnt < 8 * br.pad || br.cnt - 8 * br.pad >= 8) return CRNN_JPEG_BAD_DATA;
  for (int64_t q = br.pos; q < seg_end; ++q)
    if (f[q] != 0xFF || f[q + 1] == 0) return CRNN_JPEG_BAD_DATA;
  return CRNN_JPEG_OK;
}

// Decodes restart segment s of a 1-component scan, one block per MCU (block m of the grid is MCU m); returns a status.
__device__ __forceinline__ int decode_segment_gray(const uint8_t* f, const int64_t* seg, int s, int ri, int mcus, const HuffD& dc, const HuffD& ac,
                                   int16_t* coef) {
  const int64_t seg_end = seg[s + 1] - 2;
  BitReader br{f, seg[s], seg_end, 0ull, 0, 0};
  int pred = 0;
  const int m0 = s * ri, m1 = min(mcus, m0 + ri);
  for (int m = m0; m < m1; ++m) {
    const int e = decode_block(br, dc, ac, pred, coef + ((int64_t)m << 6));
    if (e != CRNN_JPEG_OK) return e;
    if (br.cnt < 8 * br.pad) return CRNN_JPEG_BAD_DATA;   // the segment's data ended before its MCUs
  }
  return segment_tail(f, br, seg_end);
}

// Decodes restart segment s of a 3-component interleaved scan; returns a status.  The per-component values are copied into
// arrays indexed only by unrolled constants, so they stay in registers.
__device__ __noinline__ int decode_segment_colour(const uint8_t* f, const int64_t* seg, int s, int ri, int mcus, const JGeom& g,
                                     const ParseState& ps, const HuffD* tab, uint8_t* region) {
  int H[3], V[3], bw[3], pred[3];
  int16_t* base[3];
  const HuffD* dc[3];
  const HuffD* ac[3];
#pragma unroll
  for (int sc = 0; sc < 3; ++sc) {
    const int c = ps.comp[sc];
    H[sc] = g.H[c];
    V[sc] = g.V[c];
    bw[sc] = g.bw[c];
    base[sc] = g.coef[c] >= 0 ? reinterpret_cast<int16_t*>(region + g.coef[c]) : nullptr;
    dc[sc] = &tab[ps.dct[sc]];
    ac[sc] = &tab[ps.act[sc]];
    pred[sc] = 0;
  }
  const int mcux = g.mcux;
  const int64_t seg_end = seg[s + 1] - 2;
  BitReader br{f, seg[s], seg_end, 0ull, 0, 0};
  const int m0 = s * ri, m1 = min(mcus, m0 + ri);
  for (int m = m0; m < m1; ++m) {
    const int mx = m % mcux, my = m / mcux;
#pragma unroll
    for (int sc = 0; sc < 3; ++sc)
      for (int v = 0; v < V[sc]; ++v)
        for (int u = 0; u < H[sc]; ++u) {
          int16_t* blk = base[sc] ? base[sc] + (((int64_t)(my * V[sc] + v) * bw[sc] + mx * H[sc] + u) << 6) : nullptr;
          const int e = decode_block(br, *dc[sc], *ac[sc], pred[sc], blk);
          if (e != CRNN_JPEG_OK) return e;
        }
    if (br.cnt < 8 * br.pad) return CRNN_JPEG_BAD_DATA;
  }
  return segment_tail(f, br, seg_end);
}

__global__ void __launch_bounds__(32 * JPEG_WARPS)
jpeg_entropy_kernel(const uint8_t* __restrict__ files, const int64_t* __restrict__ file_offset, const int64_t* __restrict__ file_len,
                    int N, const int* __restrict__ hs, const int* __restrict__ ws, int rule, int* __restrict__ status,
                    uint8_t* __restrict__ workspace, const int64_t* __restrict__ ws_offset, size_t bytes) {
  __shared__ WarpSmem s_warp[JPEG_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * JPEG_WARPS + warp;
  if (i >= N) return;
  WarpSmem& sm = s_warp[warp];
  ParseState& ps = sm.ps;
  const int h = hs[i], w = ws[i];
  const uint8_t* f = files + file_offset[i];
  const int64_t flen = file_len[i];
  if (lane == 0) ps.status = h < 1 || w < 1 || flen < 0 || flen > INT32_MAX ? CRNN_JPEG_BAD_HEADER : walk_markers(f, flen, h, w, rule, ps);
  __syncwarp();
  int st = ps.status;
  JGeom g;
  if (st == CRNN_JPEG_OK && !jpeg_geom(ps.sof, rule, g)) st = CRNN_JPEG_BAD_HEADER;
  if (st == CRNN_JPEG_OK && g.nf == 3) {
    if (rule == 0 && (g.H[0] != g.hmax || g.V[0] != g.vmax)) st = CRNN_JPEG_HOST_DIFFERS;   // libjpeg would upsample Y
    for (int c = 0; c < 3 && rule == 1; ++c)
      if (g.hmax % g.H[c] || g.vmax % g.V[c] || g.hmax / g.H[c] > 2 || g.vmax / g.V[c] > 2) st = CRNN_JPEG_HOST_DIFFERS;
  }
  const int64_t r0 = ws_offset[i], r1 = ws_offset[i + 1];
  if (st == CRNN_JPEG_OK && (r0 < 0 || r1 < r0 || (uint64_t)r1 > bytes || (r0 & 15) || r1 - r0 < g.bytes)) st = CRNN_JPEG_WORKSPACE;
  if (st == CRNN_JPEG_OK) {
    const int e = lane < ps.ntab ? huff_derive(f + ps.tab_pos[lane], ps.tab_dc[lane], sm.tab[lane]) : CRNN_JPEG_OK;
    st = __reduce_max_sync(0xffffffffu, e);
  }
  if (st == CRNN_JPEG_OK) {
    uint8_t* region = workspace + r0;
    JInfo* info = reinterpret_cast<JInfo*>(region);
    const int stored = g.colour ? 3 : 1;
    if (lane == 0) {
      info->colour = g.colour;
      info->ncomp = stored;
      for (int c = 0; c < 3; ++c) {
        const bool k = c < g.nf;
        info->bw[c] = k ? g.bw[c] : 0;
        info->bh[c] = k ? g.bh[c] : 0;
        info->pw[c] = k ? g.pw[c] : 0;
        info->ph[c] = k ? g.ph[c] : 0;
        info->rh[c] = k ? g.hmax / g.H[c] : 0;
        info->rv[c] = k ? g.vmax / g.V[c] : 0;
        info->coef[c] = k ? g.coef[c] : -1;
        info->plane[c] = k ? g.plane[c] : -1;
      }
    }
    for (int c = 0; c < stored; ++c)
      for (int k = lane; k < 64; k += 32) {
        const uint8_t* qv = f + (ps.qpos[c] >> 1);
        info->q[c][kNatural[k]] = (ps.qpos[c] & 1) ? (uint16_t)be16(qv + 2 * k) : qv[k];
      }
    int64_t ncoef = 0;
    for (int c = 0; c < stored; ++c) ncoef += (int64_t)g.bw[c] * g.bh[c] * 128;
    uint4* z = reinterpret_cast<uint4*>(region + g.coef[0]);
    for (int64_t k = lane; k < ncoef / 16; k += 32) z[k] = make_uint4(0, 0, 0, 0);
    // the restart segments: segment s runs from seg[s] to the marker two bytes before seg[s + 1]
    const int mcus = g.mcux * g.mcuy, ri = ps.ri ? min(ps.ri, mcus) : mcus, nseg = (mcus + ri - 1) / ri;
    int64_t* seg = reinterpret_cast<int64_t*>(region + g.segtab);
    if (lane == 0) seg[0] = ps.sos_end;
    int nrst = 0;
    int64_t eoi = -1;
    for (int64_t b0 = ps.sos_end; b0 + 1 < flen && eoi < 0 && st == CRNN_JPEG_OK; b0 += 32) {
      const int64_t p = b0 + lane;
      const bool mk = p + 1 < flen && f[p] == 0xFF && f[p + 1] != 0 && f[p + 1] != 0xFF;
      unsigned bal = __ballot_sync(0xffffffffu, mk);
      while (bal && eoi < 0 && st == CRNN_JPEG_OK) {
        const int64_t q = b0 + __ffs(bal) - 1;
        bal &= bal - 1;
        const int c = f[q + 1];
        if (c >= 0xD0 && c <= 0xD7) {
          if (c != 0xD0 + (nrst & 7) || nrst + 1 >= nseg) {
            st = CRNN_JPEG_BAD_RESTART;
          } else {
            ++nrst;
            if (lane == 0) seg[nrst] = q + 2;
          }
        } else if (c == 0xD9) {
          eoi = q;
        } else {
          st = c == 0xDA || c == 0xDC ? CRNN_JPEG_UNSUPPORTED : CRNN_JPEG_BAD_MARKER;   // a second scan, DNL, anything else
        }
      }
    }
    if (st == CRNN_JPEG_OK && eoi < 0) st = CRNN_JPEG_BAD_MARKER;
    if (st == CRNN_JPEG_OK && nrst != nseg - 1) st = CRNN_JPEG_BAD_RESTART;
    if (st == CRNN_JPEG_OK && lane == 0) seg[nseg] = eoi + 2;
    __syncwarp();
    if (st == CRNN_JPEG_OK) {
      unsigned first = 0xFFFFFFFFu;                // (segment << 4) | status of this lane's first failing segment
      for (int s = lane; s < nseg && first == 0xFFFFFFFFu; s += 32) {
        const int e = g.nf == 1 ? decode_segment_gray(f, seg, s, ri, mcus, sm.tab[ps.dct[0]], sm.tab[ps.act[0]],
                                                      reinterpret_cast<int16_t*>(region + g.coef[0]))
                                : decode_segment_colour(f, seg, s, ri, mcus, g, ps, sm.tab, region);
        if (e != CRNN_JPEG_OK) first = ((unsigned)s << 4) | (unsigned)e;
      }
      first = __reduce_min_sync(0xffffffffu, first);
      if (first != 0xFFFFFFFFu) st = (int)(first & 15);
    }
  }
  if (lane == 0) status[i] = st;
}

// ---- ISLOW: jidctint.c's constants, DESCALE and range limit.  jidctint.c computes in JLONG; here the butterflies run in 32 bits,
// which is exact because every butterfly input lies in [-ENVELOPE, ENVELOPE] (an input outside refuses its block and is replaced
// by 0): each intermediate is a fixed linear form of the 8 inputs, and the largest, sum |coefficient| x 16383, is 1.003e9 < 2^31.
constexpr int CONST_BITS = 13, PASS1_BITS = 2;
constexpr int FIX_0_298631336 = 2446, FIX_0_390180644 = 3196, FIX_0_541196100 = 4433, FIX_0_765366865 = 6270,
              FIX_0_899976223 = 7373, FIX_1_175875602 = 9633, FIX_1_501321110 = 12299, FIX_1_847759065 = 15137,
              FIX_1_961570560 = 16069, FIX_2_053119869 = 16819, FIX_2_562915447 = 20995, FIX_3_072711026 = 25172;
__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }
// IDCT_range_limit[x & RANGE_MASK]: the post-IDCT half of jdmaster.c's sample_range_limit table
__device__ __forceinline__ uint8_t range_limit(int x) {
  const int k = x & 1023;
  return (uint8_t)(k < 128 ? k + 128 : k < 512 ? 255 : k < 896 ? 0 : k - 896);
}
__device__ __forceinline__ bool outside(int v) { return v < -ENVELOPE || v > ENVELOPE; }

// The even / odd butterflies shared by both passes: in[0..7] -> out[0..7] before the descale.
__device__ __forceinline__ void islow_1d(const int* in, int* o) {
  int z2 = in[2], z3 = in[6];
  int z1 = (z2 + z3) * FIX_0_541196100;
  int tmp2 = z1 + z3 * -FIX_1_847759065, tmp3 = z1 + z2 * FIX_0_765366865;
  z2 = in[0];
  z3 = in[4];
  int tmp0 = (z2 + z3) * (1 << CONST_BITS), tmp1 = (z2 - z3) * (1 << CONST_BITS);
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = in[7];
  tmp1 = in[5];
  tmp2 = in[3];
  tmp3 = in[1];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  int z4 = tmp1 + tmp3;
  const int z5 = (z3 + z4) * FIX_1_175875602;
  tmp0 *= FIX_0_298631336;
  tmp1 *= FIX_2_053119869;
  tmp2 *= FIX_3_072711026;
  tmp3 *= FIX_1_501321110;
  z1 *= -FIX_0_899976223;
  z2 *= -FIX_2_562915447;
  z3 = z3 * -FIX_1_961570560 + z5;
  z4 = z4 * -FIX_0_390180644 + z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  o[0] = tmp10 + tmp3;
  o[7] = tmp10 - tmp3;
  o[1] = tmp11 + tmp2;
  o[6] = tmp11 - tmp2;
  o[2] = tmp12 + tmp1;
  o[5] = tmp12 - tmp1;
  o[3] = tmp13 + tmp0;
  o[4] = tmp13 - tmp0;
}

constexpr int IDCT_THREADS = 128;                  // 16 blocks at a time, 8 threads each
__global__ void __launch_bounds__(IDCT_THREADS)
jpeg_idct_kernel(int N, const int* __restrict__ hs, const int* __restrict__ ws, const int64_t* __restrict__ out_offset,
                 uint8_t* __restrict__ out, int* status, uint8_t* __restrict__ workspace, const int64_t* __restrict__ ws_offset) {
  __shared__ int s_ws[IDCT_THREADS / 8][64];
  const int i = blockIdx.x / JPEG_SPLIT, part = blockIdx.x % JPEG_SPLIT;
  if (i >= N || status[i] != CRNN_JPEG_OK) return;
  uint8_t* region = workspace + ws_offset[i];
  const JInfo* info = reinterpret_cast<const JInfo*>(region);
  const int h = hs[i], w = ws[i], colour = info->colour;
  uint8_t* dst = out + out_offset[i];
  int64_t nb[3] = {0, 0, 0}, total = 0;
  for (int c = 0; c < info->ncomp; ++c) total += nb[c] = (int64_t)info->bw[c] * info->bh[c];
  const int t = threadIdx.x & 7, lb = threadIdx.x >> 3;
  int* wsb = s_ws[lb];
  bool bad = false;
  for (int64_t b0 = (int64_t)part * (IDCT_THREADS / 8); b0 < total; b0 += (int64_t)JPEG_SPLIT * (IDCT_THREADS / 8)) {
    int64_t b = b0 + lb;
    const bool active = b < total;
    int c = 0, bw = 1, bx = 0, by = 0;
    if (active) {
      while (c < 2 && b >= nb[c]) b -= nb[c++];
      bw = info->bw[c];
      bx = (int)(b % bw);
      by = (int)(b / bw);
    }
    if (active) {                                  // pass 1: column t
      const int16_t* cf = reinterpret_cast<const int16_t*>(region + info->coef[c]) + (b << 6);
      const uint16_t* q = info->q[c];
      int in[8], o[8];
      bool ac = false;
      for (int r = 0; r < 8; ++r) {
        in[r] = cf[r * 8 + t];
        ac |= r > 0 && in[r] != 0;
      }
      if (!ac) {                                   // AC terms all zero: the column is its DC term
        const int dc = in[0] * q[t];               // |int16 x uint16| < 2^31
        const int v = dc * (1 << PASS1_BITS);
        const bool out_ = outside(dc) || outside(v);
        bad |= out_;
        for (int r = 0; r < 8; ++r) wsb[r * 8 + t] = out_ ? 0 : v;
      } else {
        for (int r = 0; r < 8; ++r) {
          in[r] *= q[r * 8 + t];
          if (outside(in[r])) {
            bad = true;
            in[r] = 0;
          }
        }
        islow_1d(in, o);
        for (int r = 0; r < 8; ++r) {
          const int v = descale(o[r], CONST_BITS - PASS1_BITS);
          bad |= outside(v);
          wsb[r * 8 + t] = outside(v) ? 0 : v;     // pass 2's inputs stay inside the envelope too
        }
      }
    }
    __syncwarp();
    if (active) {                                  // pass 2: row t
      int in[8], o[8];
      bool ac = false;
      for (int j = 0; j < 8; ++j) {
        in[j] = wsb[t * 8 + j];
        ac |= j > 0 && in[j] != 0;
      }
      if (!ac) {
        const int v = descale(in[0], PASS1_BITS + 3);
        for (int j = 0; j < 8; ++j) o[j] = v;
      } else {
        islow_1d(in, o);
        for (int j = 0; j < 8; ++j) o[j] = descale(o[j], CONST_BITS + PASS1_BITS + 3);
      }
      uint8_t px[8];
      for (int j = 0; j < 8; ++j) {
        bad |= o[j] < -512 || o[j] > 511;
        px[j] = range_limit(o[j]);
      }
      const int y = by * 8 + t;
      if (colour) {
        uint8_t* row = region + info->plane[c] + (int64_t)y * bw * 8 + bx * 8;
        *reinterpret_cast<uint2*>(row) = make_uint2(px[0] | px[1] << 8 | px[2] << 16 | (uint32_t)px[3] << 24,
                                                    px[4] | px[5] << 8 | px[6] << 16 | (uint32_t)px[7] << 24);
      } else if (y < h) {
        for (int j = 0; j < 8 && bx * 8 + j < w; ++j) dst[(int64_t)y * w + bx * 8 + j] = px[j];
      }
    }
    __syncwarp();
  }
  if (bad) status[i] = CRNN_JPEG_HOST_DIFFERS;     // every writer stores the same value; the finish kernel zeroes the slot
}

// Sample (x, y) of component c upsampled to the output grid: libjpeg-turbo's jdsample.c for the ratios rule 1 reads.
__device__ __forceinline__ int upsample(const JInfo* info, const uint8_t* region, int c, int x, int y) {
  const uint8_t* P = region + info->plane[c];
  const int64_t stride = (int64_t)info->bw[c] * 8;
  const int rh = info->rh[c], rv = info->rv[c], dw = info->pw[c], dh = info->ph[c];
  if (rh == 1 && rv == 1) return P[y * stride + x];
  const int j = x >> 1, r = y >> 1;
  if (rv == 1) {                                   // h2v1: fancy when the component is more than 2 samples wide
    const uint8_t* row = P + y * stride;
    if (dw <= 2) return row[j];
    if (x & 1) return j == dw - 1 ? row[j] : (3 * row[j] + row[j + 1] + 2) >> 2;
    return j == 0 ? row[0] : (3 * row[j] + row[j - 1] + 1) >> 2;
  }
  const int nbr = (y & 1) ? min(r + 1, dh - 1) : max(r - 1, 0);   // the edge rows repeat themselves
  const uint8_t* r0 = P + r * stride;
  const uint8_t* r1 = P + nbr * stride;
  if (rh == 1) return (3 * r0[x] + r1[x] + ((y & 1) ? 2 : 1)) >> 2;   // h1v2: biases 1 above, 2 below
  if (dw <= 2) return r0[j];                       // h2v2 box
  const int cs = 3 * r0[j] + r1[j];
  if (x & 1) return j == dw - 1 ? (cs * 4 + 7) >> 4 : (3 * cs + 3 * r0[j + 1] + r1[j + 1] + 7) >> 4;
  return j == 0 ? (cs * 4 + 8) >> 4 : (3 * cs + 3 * r0[j - 1] + r1[j - 1] + 8) >> 4;
}

constexpr int FINISH_THREADS = 256;
__global__ void __launch_bounds__(FINISH_THREADS)
jpeg_finish_kernel(int N, const int* __restrict__ hs, const int* __restrict__ ws, const int64_t* __restrict__ out_offset,
                   uint8_t* __restrict__ out, const int* __restrict__ status, const uint8_t* __restrict__ workspace,
                   const int64_t* __restrict__ ws_offset) {
  const int i = blockIdx.x / JPEG_SPLIT, part = blockIdx.x % JPEG_SPLIT;
  if (i >= N) return;
  const int h = hs[i], w = ws[i];
  if (h < 1 || w < 1) return;
  uint8_t* dst = out + out_offset[i];
  const int64_t n = (int64_t)h * w, step = (int64_t)JPEG_SPLIT * FINISH_THREADS;
  if (status[i] != CRNN_JPEG_OK) {
    for (int64_t p = (int64_t)part * FINISH_THREADS + threadIdx.x; p < n; p += step) dst[p] = 0;
    return;
  }
  const uint8_t* region = workspace + ws_offset[i];
  const JInfo* info = reinterpret_cast<const JInfo*>(region);
  if (!info->colour) return;
  for (int64_t p = (int64_t)part * FINISH_THREADS + threadIdx.x; p < n; p += step) {
    const int y = (int)(p / w), x = (int)(p - (int64_t)y * w);
    const int Y = upsample(info, region, 0, x, y), cb = upsample(info, region, 1, x, y) - 128, cr = upsample(info, region, 2, x, y) - 128;
    // jdcolor.c's Cr_r / Cb_b / Cr_g / Cb_g tables (SCALEBITS 16), then the sample range limit
    const int R = min(max(Y + ((91881 * cr + 32768) >> 16), 0), 255);
    const int G = min(max(Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16), 0), 255);
    const int B = min(max(Y + ((116130 * cb + 32768) >> 16), 0), 255);
    dst[p] = (uint8_t)((19595 * R + 38470 * G + 7471 * B + 0x8000) >> 16);
  }
}

}  // namespace

extern "C" int crnn_jpeg_plan(const uint8_t* sof, const int64_t* file_len, int N, int rule, int64_t* ws_offset, size_t* workspace_bytes) {
  if (!sof || !file_len || !ws_offset || !workspace_bytes) return crnn_fail(CRNN_INVALID_VALUE, "jpeg_plan: null pointer");
  if (N <= 0) return crnn_fail(CRNN_INVALID_VALUE, "jpeg_plan: N = %d", N);
  if (rule != 0 && rule != 1) return crnn_fail(CRNN_INVALID_VALUE, "jpeg_plan: rule = %d (0: OpenCV, 1: Pillow)", rule);
  int64_t off = 0;
  for (int i = 0; i < N; ++i) {
    ws_offset[i] = off;
    JGeom g;
    if (file_len[i] > 0 && jpeg_geom(sof + 16 * (size_t)i, rule, g)) off += g.bytes;
  }
  ws_offset[N] = off;
  *workspace_bytes = (size_t)off;
  return CRNN_OK;
}

extern "C" int crnn_jpeg_decode_gray_u8(const uint8_t* files, const int64_t* file_offset, const int64_t* file_len, int N, const int* h,
                                        const int* w, const int64_t* out_offset, int rule, uint8_t* out, int* status, void* workspace,
                                        const int64_t* ws_offset, size_t bytes, crnn_stream_t stream) {
  static const char* fn = "jpeg_decode_gray_u8";
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
  CRNN_TRY(check_aligned(workspace, 16, fn, "workspace"));
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* wsp = static_cast<uint8_t*>(workspace);
  jpeg_entropy_kernel<<<(N + JPEG_WARPS - 1) / JPEG_WARPS, 32 * JPEG_WARPS, 0, s>>>(files, file_offset, file_len, N, h, w, rule, status,
                                                                                   wsp, ws_offset, bytes);
  CUDA_TRY(cudaGetLastError());
  const unsigned grid = (unsigned)N * JPEG_SPLIT;
  jpeg_idct_kernel<<<grid, IDCT_THREADS, 0, s>>>(N, h, w, out_offset, out, status, wsp, ws_offset);
  CUDA_TRY(cudaGetLastError());
  jpeg_finish_kernel<<<grid, FINISH_THREADS, 0, s>>>(N, h, w, out_offset, out, status, wsp, ws_offset);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
