// Training lines rendered on the device, sm_90a: a counter-based layout stream, glyphs composited into 60-row canvases with
// Pillow's blend arithmetic, and resize.cu's Pillow BILINEAR resize to the [N, W, 32] uint8 batch groupBatch builds.
//
// Random stream: Philox4x64-10 (Salmon et al., SC'11), key = (seed, RD_KEY1), counter = (line, attempt, block, 0); one call
// gives a block of four 64-bit words w0..w3.  numpy's np.random.Philox is the same cipher (it increments its counter before
// each block, so its first block for counter c is philox(c + 1)).  An integer in [a, b] is a + ((u * (b - a + 1)) >> 64) from
// one word u: the count of u giving each value differs by at most one, a bias below (b - a + 1) / 2^64 < 2^-57 for every
// range drawn here.  Word order of line i, attempt t (restated by gen.philox_layout):
//   block 0       w0 length U[min_len, max_len]   w1 background U[180, 255]   w2 x0 U[2, 12]     (w3 unused)
//   block 1 + j   w0 glyph j's charset index U[0, nglyphs - 1]   w1 y U[0, 10]   w2 fill U[0, 90]   w3 advance jitter U[-2, 3]
// render_line's layout (lib/lstm/utils/gen.py): glyph j is drawn at (x_j, y_j), x_0 = x0, x_{j+1} = x_j + adv_j + dx_j, on a
// 60 x (sum adv + 28) canvas; the resized width is nw = (int)(32.0 / 60 * canvas_w) in double, time_step = nw / 4 - 1.
// A bucketed stream (nw_hi > 0) redraws line i with attempt t + 1 until nw_lo < nw <= nw_hi, at most RD_MAX_ATTEMPTS times.
//
// render_layout_kernel: one CTA, one thread per line in chunks of RL_THREADS; the flat label offsets are a block-wide prefix sum.
// render_composite_kernel: one CTA per (line, tile of 32 canvas columns).  The glyphs meeting the tile are listed in draw order
// in shared memory; each thread then owns pixels (row, column): background, then every listed glyph whose mask covers the pixel,
// blended as Pillow's fill_mask_L (ImagingFill2 behind ImageDraw's draw_bitmap):
//   out = DIV255(out * (255 - m) + fill * m),  DIV255(v) = (((v + 128) >> 8) + v + 128) >> 8
// Pixels outside the canvas are never visited, which is the clipping ImagingFill2 applies on all four sides.
#include "common.cuh"
#include "resize.h"
#include <stdint.h>

namespace {

constexpr int RD_ROWS = 60;                // canvas height (render_line's)
constexpr int RD_MARGIN = 28;              // canvas width beyond the glyph advances
constexpr int RD_HDR = 8;                  // ints of a layout record before its per-glyph arrays
constexpr int RD_MAX_CHARS = 256;          // characters per line
constexpr int RD_MAX_GLYPHS = 62;          // charset size (label ids 1 .. 62)
constexpr int RD_MAX_ATTEMPTS = 256;       // redraws of a bucketed line before the call reports the bucket unreachable
constexpr int RD_GLYPH_INTS = 8;           // glyph table row: adv, w, h, ox, oy, mask offset, 0, 0
constexpr uint64_t RD_KEY1 = 0x43524e4e52454e44ull;   // "CRNNREND"
constexpr int RL_THREADS = 256, RL_WARPS = RL_THREADS / 32;
constexpr int RC_TILE = 32, RC_THREADS = 256;

struct Words { uint64_t w[4]; };

__device__ __forceinline__ Words philox4x64_10(uint64_t c0, uint64_t c1, uint64_t c2, uint64_t c3, uint64_t k0, uint64_t k1) {
  constexpr uint64_t M0 = 0xD2E7470EE14C6C93ull, M1 = 0xCA5A826395121157ull;
  constexpr uint64_t W0 = 0x9E3779B97F4A7C15ull, W1 = 0xBB67AE8584CAA73Bull;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += W0; k1 += W1; }
    const uint64_t hi0 = __umul64hi(M0, c0), lo0 = M0 * c0;
    const uint64_t hi1 = __umul64hi(M1, c2), lo1 = M1 * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
  }
  Words out;
  out.w[0] = c0; out.w[1] = c1; out.w[2] = c2; out.w[3] = c3;
  return out;
}

__device__ __forceinline__ int rd_draw(uint64_t u, int a, int b) { return a + (int)__umul64hi(u, (uint64_t)(b - a + 1)); }

// Block-wide exclusive prefix sum of v over the RL_THREADS threads; *total gets the sum.  s_ws holds RL_WARPS + 1 ints.
__device__ __forceinline__ int rl_block_scan(int v, int* s_ws, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_ws[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = lane < RL_WARPS ? s_ws[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    if (lane < RL_WARPS) s_ws[lane + 1] = w;
    if (lane == 0) s_ws[0] = 0;
  }
  __syncthreads();
  const int out = s_ws[warp] + x - v;
  *total = s_ws[RL_WARPS];
  __syncthreads();                       // s_ws is reused by the next call
  return out;
}

// layout record of a line ([N][RD_HDR + 4 * max_len] i32):
//   [0] length  [1] background  [2] x0  [3] canvas width  [4] nw  [5] time_step  [6] flat label offset  [7] attempt
//   then chars (label ids 1 .. nglyphs) [max_len], x [max_len], y [max_len], fill [max_len]
// feeds ([4 + 2N + N * max_len] i32): [0] lines that found no width in the bucket  [1] max nw  [2] labels in total
//   [3] padded width W   then label_len [N], time_step [N], flat labels
__global__ void __launch_bounds__(RL_THREADS)
render_layout_kernel(uint64_t seed, int N, int min_len, int max_len, int nw_lo, int nw_hi, const int* __restrict__ glyphs,
                     int nglyphs, int* __restrict__ layout, int* __restrict__ feeds) {
  __shared__ int s_adv[RD_MAX_GLYPHS];
  __shared__ int s_ws[RL_WARPS + 1];
  __shared__ int s_maxnw, s_fail;
  const int tid = threadIdx.x;
  if (tid < nglyphs) s_adv[tid] = glyphs[tid * RD_GLYPH_INTS];
  if (tid == 0) { s_maxnw = 0; s_fail = 0; }
  __syncthreads();
  const size_t rec_stride = RD_HDR + 4 * (size_t)max_len;
  int* lab_len = feeds + 4;
  int* tsl_out = lab_len + N;
  int* labels = tsl_out + N;
  int carry = 0;
  for (int base = 0; base < N; base += RL_THREADS) {
    const int i = base + tid;
    int len = 0;
    int* rec = layout + (size_t)i * rec_stride;
    if (i < N) {
      int attempt = 0, bg = 0, x0 = 0, cw = 0, nw = 0;
      for (;; ++attempt) {
        const Words b0 = philox4x64_10((uint64_t)i, (uint64_t)attempt, 0, 0, seed, RD_KEY1);
        len = rd_draw(b0.w[0], min_len, max_len);
        bg = rd_draw(b0.w[1], 180, 255);
        x0 = rd_draw(b0.w[2], 2, 12);
        int x = x0;
        cw = RD_MARGIN;
        for (int j = 0; j < len; ++j) {
          const Words b = philox4x64_10((uint64_t)i, (uint64_t)attempt, (uint64_t)(1 + j), 0, seed, RD_KEY1);
          const int c = rd_draw(b.w[0], 0, nglyphs - 1);
          rec[RD_HDR + j] = c + 1;
          rec[RD_HDR + max_len + j] = x;
          rec[RD_HDR + 2 * max_len + j] = rd_draw(b.w[1], 0, 10);
          rec[RD_HDR + 3 * max_len + j] = rd_draw(b.w[2], 0, 90);
          x += s_adv[c] + rd_draw(b.w[3], -2, 3);
          cw += s_adv[c];
        }
        nw = __double2int_rz(__dmul_rn(__ddiv_rn(32.0, (double)RD_ROWS), (double)cw));
        if (nw_hi == 0 || (nw > nw_lo && nw <= nw_hi)) break;
        if (attempt + 1 == RD_MAX_ATTEMPTS) { atomicAdd(&s_fail, 1); break; }
      }
      rec[0] = len; rec[1] = bg; rec[2] = x0; rec[3] = cw; rec[4] = nw; rec[5] = nw / 4 - 1; rec[7] = attempt;
      lab_len[i] = len;
      tsl_out[i] = nw / 4 - 1;
      atomicMax(&s_maxnw, nw);
    }
    int total;
    const int off = carry + rl_block_scan(len, s_ws, &total);
    if (i < N) {
      rec[6] = off;
      for (int j = 0; j < len; ++j) labels[off + j] = rec[RD_HDR + j];
    }
    carry += total;
  }
  __syncthreads();
  if (tid == 0) {
    feeds[0] = s_fail;
    feeds[1] = s_maxnw;
    feeds[2] = carry;
    feeds[3] = nw_hi ? nw_hi : max(8, (s_maxnw + 3) / 4 * 4);
  }
}

__device__ __forceinline__ uint32_t div255(uint32_t v) { return (((v + 128u) >> 8) + v + 128u) >> 8; }

// Workspace: src_offset i64 [N], src_h, src_w, out_w i32 [N] (the resize's tables), then N canvases of RD_ROWS x stride bytes;
// canvas i is row-major with row length canvas_w[i] at byte i * RD_ROWS * stride.
__global__ void __launch_bounds__(RC_THREADS)
render_composite_kernel(const int* __restrict__ layout, int max_len, const int* __restrict__ glyphs, const uint8_t* __restrict__ masks,
                        int stride, int64_t* __restrict__ src_off, int* __restrict__ src_h, int* __restrict__ src_w,
                        int* __restrict__ out_w, uint8_t* __restrict__ canvas) {
  __shared__ int s_sx[RD_MAX_CHARS], s_sy[RD_MAX_CHARS], s_gw[RD_MAX_CHARS], s_gh[RD_MAX_CHARS], s_fill[RD_MAX_CHARS],
      s_moff[RD_MAX_CHARS];
  __shared__ unsigned s_hit[RD_MAX_CHARS / 32];
  const int i = blockIdx.x, c0 = blockIdx.y * RC_TILE, tid = threadIdx.x;
  const int* rec = layout + (size_t)i * (RD_HDR + 4 * (size_t)max_len);
  const int len = rec[0], bg = rec[1], cw = rec[3], nw = rec[4];
  // a record the call did not write for this max_len / atlas gets an all-zero slot from the resize (src_h = 0)
  const bool ok = len >= 1 && len <= max_len && cw >= 1 && cw <= stride && nw >= 1;
  if (blockIdx.y == 0 && tid == 0) {
    src_off[i] = (int64_t)i * RD_ROWS * stride;
    src_h[i] = ok ? RD_ROWS : 0;
    src_w[i] = ok ? cw : 1;
    out_w[i] = ok ? nw : 1;
  }
  if (!ok || c0 >= cw) return;
  // the glyphs whose masks meet columns [c0, c0 + RC_TILE), in draw order
  const int* chars = rec + RD_HDR;
  int sx = 0, gw = 0, ch = 0;
  bool hit = false;
  if (tid < len) {
    ch = chars[tid] - 1;
    const int* g = glyphs + ch * RD_GLYPH_INTS;
    gw = g[1];
    sx = rec[RD_HDR + max_len + tid] + g[3];
    hit = gw > 0 && g[2] > 0 && sx < c0 + RC_TILE && sx + gw > c0;
  }
  const unsigned ballot = __ballot_sync(0xffffffffu, hit);
  if ((tid & 31) == 0 && tid < RD_MAX_CHARS) s_hit[tid >> 5] = ballot;
  __syncthreads();
  int before = 0, count = 0;
  for (int k = 0; k < (len + 31) / 32; ++k) {
    const int p = __popc(s_hit[k]);
    if (k < (tid >> 5)) before += p;
    count += p;
  }
  if (hit) {
    const int slot = before + __popc(ballot & ((1u << (tid & 31)) - 1u));
    const int* g = glyphs + ch * RD_GLYPH_INTS;
    s_sx[slot] = sx;
    s_sy[slot] = rec[RD_HDR + 2 * max_len + tid] + g[4];
    s_gw[slot] = gw;
    s_gh[slot] = g[2];
    s_fill[slot] = rec[RD_HDR + 3 * max_len + tid];
    s_moff[slot] = g[5];
  }
  __syncthreads();
  uint8_t* dst = canvas + (size_t)i * RD_ROWS * stride;
  for (int e = tid; e < RD_ROWS * RC_TILE; e += RC_THREADS) {
    const int r = e / RC_TILE, c = c0 + e % RC_TILE;
    if (c >= cw) continue;
    uint32_t v = (uint32_t)bg;
    for (int k = 0; k < count; ++k) {
      const int mx = c - s_sx[k], my = r - s_sy[k];
      if ((unsigned)mx < (unsigned)s_gw[k] && (unsigned)my < (unsigned)s_gh[k]) {
        const uint32_t m = __ldg(masks + s_moff[k] + my * s_gw[k] + mx);
        v = div255(v * (255u - m) + (uint32_t)s_fill[k] * m);
      }
    }
    dst[(size_t)r * cw + c] = (uint8_t)v;
  }
}

inline size_t rd_align(size_t b) { return (b + 255) & ~(size_t)255; }
inline int rd_stride(int max_len, int max_adv) { return max_len * max_adv + RD_MARGIN; }
inline size_t rd_workspace(int N, int max_len, int max_adv) {
  return rd_align(sizeof(int64_t) * N) + 3 * rd_align(sizeof(int) * N) + (size_t)N * RD_ROWS * rd_stride(max_len, max_adv);
}

}  // namespace

extern "C" int crnn_render_layout(int64_t seed, int N, int min_len, int max_len, int nw_lo, int nw_hi, const int* glyphs,
                                  int nglyphs, int* layout, int* feeds, crnn_stream_t stream) {
  if (!glyphs || !layout || !feeds) return crnn_fail(CRNN_INVALID_VALUE, "render_layout: null pointer");
  if (N <= 0) return crnn_fail(CRNN_INVALID_VALUE, "render_layout: N = %d", N);
  if (min_len < 1 || max_len < min_len)
    return crnn_fail(CRNN_INVALID_VALUE, "render_layout: bad length range [%d, %d]", min_len, max_len);
  if (max_len > RD_MAX_CHARS)
    return crnn_fail(CRNN_UNSUPPORTED, "render_layout: max_len = %d beyond the %d characters a line holds", max_len, RD_MAX_CHARS);
  if (nglyphs < 1 || nglyphs > RD_MAX_GLYPHS)
    return crnn_fail(CRNN_INVALID_VALUE, "render_layout: nglyphs = %d outside [1, %d]", nglyphs, RD_MAX_GLYPHS);
  if (nw_hi != 0 && (nw_hi < 8 || nw_hi % 4 || nw_lo < 0 || nw_lo >= nw_hi))
    return crnn_fail(CRNN_INVALID_VALUE, "render_layout: bad bucket (%d, %d]", nw_lo, nw_hi);
  render_layout_kernel<<<1, RL_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>((uint64_t)seed, N, min_len, max_len, nw_lo,
                                                                                    nw_hi, glyphs, nglyphs, layout, feeds);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}

extern "C" int crnn_render_workspace_size(int N, int max_len, int max_adv, size_t* bytes) {
  if (!bytes) return crnn_fail(CRNN_INVALID_VALUE, "render_workspace_size: null pointer");
  if (N <= 0 || max_len < 1 || max_adv < 1) return crnn_fail(CRNN_INVALID_VALUE, "render_workspace_size: N = %d, max_len = %d, max_adv = %d", N, max_len, max_adv);
  if (max_len > RD_MAX_CHARS)
    return crnn_fail(CRNN_UNSUPPORTED, "render_workspace_size: max_len = %d beyond the %d characters a line holds", max_len, RD_MAX_CHARS);
  if ((size_t)rd_stride(max_len, max_adv) > (size_t)65535 * RC_TILE)
    return crnn_fail(CRNN_UNSUPPORTED, "render_workspace_size: canvases of %d columns are beyond the kernel", rd_stride(max_len, max_adv));
  *bytes = rd_workspace(N, max_len, max_adv);
  return CRNN_OK;
}

extern "C" int crnn_render_lines_u8(const int* layout, int N, int max_len, const int* glyphs, const uint8_t* masks, int max_adv,
                                    int W, void* workspace, size_t workspace_bytes, uint8_t* out, crnn_stream_t stream) {
  if (!layout || !glyphs || !masks || !workspace || !out) return crnn_fail(CRNN_INVALID_VALUE, "render_lines_u8: null pointer");
  if (N <= 0 || max_len < 1 || max_adv < 1 || W < 8 || W % 4)
    return crnn_fail(CRNN_INVALID_VALUE, "render_lines_u8: bad shape N = %d, max_len = %d, max_adv = %d, W = %d (W a multiple of 4, >= 8)",
                     N, max_len, max_adv, W);
  if (reinterpret_cast<uintptr_t>(out) & 3 || reinterpret_cast<uintptr_t>(workspace) & 255)
    return crnn_fail(CRNN_INVALID_VALUE, "render_lines_u8: out must be 4-byte and workspace 256-byte aligned");
  if (max_len > RD_MAX_CHARS)
    return crnn_fail(CRNN_UNSUPPORTED, "render_lines_u8: max_len = %d beyond the %d characters a line holds", max_len, RD_MAX_CHARS);
  const int stride = rd_stride(max_len, max_adv);
  if ((W + 31) / 32 > 65535 || (stride + RC_TILE - 1) / RC_TILE > 65535)
    return crnn_fail(CRNN_UNSUPPORTED, "render_lines_u8: W = %d or canvases of %d columns beyond the kernels", W, stride);
  if (workspace_bytes < rd_workspace(N, max_len, max_adv))
    return crnn_fail(CRNN_WORKSPACE_TOO_SMALL, "render_lines_u8: workspace of %zu bytes, %zu needed", workspace_bytes,
                     rd_workspace(N, max_len, max_adv));
  char* ws = static_cast<char*>(workspace);
  int64_t* src_off = reinterpret_cast<int64_t*>(ws);
  int* src_h = reinterpret_cast<int*>(ws + rd_align(sizeof(int64_t) * N));
  int* src_w = reinterpret_cast<int*>(reinterpret_cast<char*>(src_h) + rd_align(sizeof(int) * N));
  int* out_w = reinterpret_cast<int*>(reinterpret_cast<char*>(src_w) + rd_align(sizeof(int) * N));
  uint8_t* canvas = reinterpret_cast<uint8_t*>(out_w) + rd_align(sizeof(int) * N);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  render_composite_kernel<<<dim3(N, (stride + RC_TILE - 1) / RC_TILE), RC_THREADS, 0, st>>>(layout, max_len, glyphs, masks, stride,
                                                                                            src_off, src_h, src_w, out_w, canvas);
  CUDA_TRY(cudaGetLastError());
  return resize_lines_u8_launch(canvas, src_off, src_h, src_w, out_w, N, W, RD_ROWS, out, st);
}
