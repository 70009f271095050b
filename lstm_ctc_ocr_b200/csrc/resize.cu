// Resize native-size 8-bit gray text lines to the network's 32 rows, sm_90a: byte for byte Pillow's
// Image.resize((out_w, 32), Image.BILINEAR) on mode "L", written width-major into a packed [N, W, 32] u8 batch.
//
// Pillow's 8-bit BILINEAR (Resample.c: precompute_coeffs, normalize_coeffs_8bpc, ImagingResample{Horizontal,Vertical}_8bpc) for
// one axis, in_size -> out_size, PB = 22:
//   scale = in / out;  fs = max(scale, 1);  support = fs;  ss = 1 / fs
//   center = (xx + 0.5) * scale;  xmin = max(0, (int)(center - support + 0.5));  n = min(in, (int)(center + support + 0.5)) - xmin
//   w[x] = max(0, 1 - |(x + xmin - center + 0.5) * ss|), ww = sum w in order, w[x] /= ww (ww != 0), k[x] = (int)(w[x] * 2^PB + 0.5)
//   out[xx] = clamp((2^(PB-1) + sum src[xmin + x] * k[x]) >> PB, 0, 255)      (int32 accumulator)
// The horizontal pass (w -> out_w) runs on every row first, the vertical pass (h -> 32) on its u8 result; a pass whose size is
// unchanged is skipped.  A source more than 100 times taller than wide (h > 100 w) takes the passes the other way round, vertical
// first, as Pillow 12 does; under the evaluation size rule that is a line of 2 .. 10 columns resized to out_w = 1.
// The coefficients are double arithmetic through __d*_rn intrinsics, so no product is contracted into an FMA: 1 - |(...) * ss| or
// w * 2^PB + 0.5 as an FMA would round differently from Pillow's compiled C and change the weights.
//
// resize_lines_u8_kernel: one CTA per (line, tile of 32 output columns).
//   coefficients  warp 0: one thread per output column of the tile (horizontal); warp 1: one thread per output row (vertical),
//                 into shared memory; tables sized from max_h (a line's taps: 2 * ceil(support) + 1)
//   horizontal    thread = (source row, column of the tile) -> the h x 32 u8 intermediate in shared memory
//   vertical      thread = (column, 4 output rows): one 4-byte store, so a warp writes 4 whole 32-byte columns
//   (h > 100 w: the vertical pass on the source's w < h / 100 columns into a 32 x w intermediate, then the horizontal pass
//    from it in the store loop)
// Columns from out_w[i] to W are written as zero, so the batch needs no memset.
#include "common.cuh"
#include "resize.h"
#include <stdint.h>

namespace {

constexpr int RS_TILE = 32;          // output columns per CTA
constexpr int RS_THREADS = 256;
constexpr int RS_OUT_H = 32;         // cfg.IMG_HEIGHT
constexpr int RS_MAX_H = 1024;       // tallest source line: its intermediate (max_h x 32 bytes) and tap tables stay in shared memory
constexpr int RS_PB = 22;            // Pillow's PRECISION_BITS for 8-bit images

// Taps per output position of the tables, from the tallest line.  Vertical: support = max(h / 32, 1).  Horizontal under the size
// rule out_w = max(1, (int)(32 / h * w)): w / out_w < h / 16 (+ rounding), so ceil(support) <= ceil(max_h / 16) + 1.
__host__ __device__ inline int rs_kh_cap(int max_h) { return 2 * ((max_h + 15) / 16 + 1) + 1; }
__host__ __device__ inline int rs_kv_cap(int max_h) { return 2 * ((max_h + 31) / 32) + 1; }
inline size_t rs_smem_bytes(int max_h) {
  return sizeof(int) * (size_t)(RS_TILE * rs_kh_cap(max_h) + RS_OUT_H * rs_kv_cap(max_h)) + (size_t)max_h * RS_TILE;
}

__device__ __forceinline__ double rs_scale(int in_size, int out_size) { return __ddiv_rn((double)in_size, (double)out_size); }

// Pillow's ksize: 2 * ceil(support) + 1 taps hold every output position's window.
__device__ __forceinline__ int rs_ksize(int in_size, int out_size) {
  const double s = rs_scale(in_size, out_size);
  return 2 * (int)ceil(s < 1.0 ? 1.0 : s) + 1;
}

__device__ __forceinline__ double rs_tap(int x, double center, double ss) {   // bilinear_filter((x + xmin - center + 0.5) * ss)
  double t = __dmul_rn(__dadd_rn(__dsub_rn((double)x, center), 0.5), ss);
  t = fabs(t);
  return t < 1.0 ? __dsub_rn(1.0, t) : 0.0;
}

// The integer taps of output position xx; returns n, writes xmin.  n <= rs_ksize(in_size, out_size).
__device__ int rs_coeffs(int in_size, int out_size, int xx, int* __restrict__ k, int* __restrict__ xmin_out) {
  const double scale = rs_scale(in_size, out_size);
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double support = fs;                         // bilinear support 1.0 times the filter scale
  const double ss = __ddiv_rn(1.0, fs);
  const double center = __dmul_rn(__dadd_rn((double)xx, 0.5), scale);
  int xmin = __double2int_rz(__dadd_rn(__dsub_rn(center, support), 0.5));
  if (xmin < 0) xmin = 0;
  int xmax = __double2int_rz(__dadd_rn(__dadd_rn(center, support), 0.5));
  if (xmax > in_size) xmax = in_size;
  const int n = xmax - xmin;
  double ww = 0.0;
  for (int x = 0; x < n; ++x) ww = __dadd_rn(ww, rs_tap(x + xmin, center, ss));
  for (int x = 0; x < n; ++x) {
    double w = rs_tap(x + xmin, center, ss);
    if (ww != 0.0) w = __ddiv_rn(w, ww);
    k[x] = __double2int_rz(w < 0.0 ? __dadd_rn(__dmul_rn(w, (double)(1 << RS_PB)), -0.5) : __dadd_rn(__dmul_rn(w, (double)(1 << RS_PB)), 0.5));
  }
  *xmin_out = xmin;
  return n;
}

__device__ __forceinline__ uint32_t rs_clip8(int acc) {
  const int v = acc >> RS_PB;
  return (uint32_t)(v < 0 ? 0 : v > 255 ? 255 : v);
}

__global__ void __launch_bounds__(RS_THREADS)
resize_lines_u8_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ src_offset, const int* __restrict__ src_h,
                       const int* __restrict__ src_w, const int* __restrict__ out_w, int W, int max_h, uint8_t* __restrict__ out) {
  extern __shared__ __align__(16) int rs_smem[];
  __shared__ int s_xmin[RS_TILE], s_xn[RS_TILE], s_ymin[RS_OUT_H], s_yn[RS_OUT_H];
  const int kh_cap = rs_kh_cap(max_h), kv_cap = rs_kv_cap(max_h);
  int* s_kh = rs_smem;                                                       // [RS_TILE][kh_cap] horizontal taps
  int* s_kv = s_kh + RS_TILE * kh_cap;                                       // [32][kv_cap] vertical taps
  uint8_t* s_mid = reinterpret_cast<uint8_t*>(s_kv + RS_OUT_H * kv_cap);     // [h][RS_TILE] horizontal pass result

  const int i = blockIdx.x, x0 = blockIdx.y * RS_TILE, tid = threadIdx.x;
  const int cols = min(RS_TILE, W - x0);
  const int h = src_h[i], w = src_w[i], nw = out_w[i];
  const bool need_h = nw != w, need_v = h != RS_OUT_H;
  const bool v_first = need_h && need_v && h > 100 * w;                     // Pillow's order for tall, narrow sources
  // a line outside the preconditions gets an all-zero slot and is never read
  const bool ok = h >= 1 && h <= max_h && w >= 1 && nw >= 1 && (!need_h || rs_ksize(w, nw) <= kh_cap) &&
                  (!need_v || rs_ksize(h, RS_OUT_H) <= kv_cap);
  const int valid = ok ? max(0, min(cols, nw - x0)) : 0;                     // columns of this tile inside the line
  uint32_t* dst = reinterpret_cast<uint32_t*>(out + ((size_t)i * W + x0) * RS_OUT_H);
  if (valid == 0) {                                                          // padding only
    for (int e = tid; e < cols * (RS_OUT_H / 4); e += RS_THREADS) dst[e] = 0u;
    return;
  }
  const uint8_t* img = src + src_offset[i];
  if (need_h && tid < valid) s_xn[tid] = rs_coeffs(w, nw, x0 + tid, s_kh + tid * kh_cap, &s_xmin[tid]);
  if (need_v && tid >= 32 && tid < 32 + RS_OUT_H) {
    const int y = tid - 32;
    s_yn[y] = rs_coeffs(h, RS_OUT_H, y, s_kv + y * kv_cap, &s_ymin[y]);
  }
  __syncthreads();

  if (v_first) {                                                            // 32 x w intermediate, row stride w (< h / 100)
    for (int e = tid; e < RS_OUT_H * w; e += RS_THREADS) {
      const int y = e / w, c = e - y * w;
      const int* k = s_kv + y * kv_cap;
      const uint8_t* p = img + (size_t)s_ymin[y] * w + c;
      const int n = s_yn[y];
      int acc = 1 << (RS_PB - 1);
      for (int j = 0; j < n; ++j) acc += (int)__ldg(p + (size_t)j * w) * k[j];
      s_mid[e] = (uint8_t)rs_clip8(acc);
    }
  }
  for (int e = tid; e < (v_first ? 0 : h * valid); e += RS_THREADS) {
    const int y = e / valid, c = e - y * valid;
    const uint8_t* row = img + (size_t)y * w;
    uint32_t v;
    if (need_h) {
      const int* k = s_kh + c * kh_cap;
      const uint8_t* p = row + s_xmin[c];
      const int n = s_xn[c];
      int acc = 1 << (RS_PB - 1);
      for (int x = 0; x < n; ++x) acc += (int)__ldg(p + x) * k[x];
      v = rs_clip8(acc);
    } else {
      v = __ldg(row + x0 + c);
    }
    s_mid[y * RS_TILE + c] = (uint8_t)v;
  }
  __syncthreads();

  for (int e = tid; e < cols * (RS_OUT_H / 4); e += RS_THREADS) {
    const int c = e >> 3, y0 = (e & 7) * 4;
    uint32_t word = 0u;
    if (c < valid) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int y = y0 + r;
        uint32_t v;
        if (v_first) {
          const int* k = s_kh + c * kh_cap;
          const uint8_t* p = s_mid + y * w + s_xmin[c];
          const int n = s_xn[c];
          int acc = 1 << (RS_PB - 1);
          for (int x = 0; x < n; ++x) acc += (int)p[x] * k[x];
          v = rs_clip8(acc);
        } else if (need_v) {
          const int* k = s_kv + y * kv_cap;
          const uint8_t* p = s_mid + s_ymin[y] * RS_TILE + c;
          const int n = s_yn[y];
          int acc = 1 << (RS_PB - 1);
          for (int j = 0; j < n; ++j) acc += (int)p[j * RS_TILE] * k[j];
          v = rs_clip8(acc);
        } else {
          v = s_mid[y * RS_TILE + c];
        }
        word |= v << (8 * r);
      }
    }
    dst[e] = word;                       // bytes y0 .. y0+3 of column x0 + c
  }
}

}  // namespace

int resize_lines_u8_launch(const uint8_t* src, const int64_t* src_offset, const int* src_h, const int* src_w, const int* out_w,
                           int N, int W, int max_h, uint8_t* out, cudaStream_t stream) {
  const int tiles = (W + RS_TILE - 1) / RS_TILE;
  const size_t smem = rs_smem_bytes(max_h);
  if (smem > 48 * 1024)
    CUDA_TRY(cudaFuncSetAttribute(resize_lines_u8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  resize_lines_u8_kernel<<<dim3(N, tiles), RS_THREADS, smem, stream>>>(src, src_offset, src_h, src_w, out_w, W, max_h, out);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}

extern "C" int crnn_resize_lines_u8(const uint8_t* src, const int64_t* src_offset, const int* src_h, const int* src_w,
                                    const int* out_w, int N, int W, int max_h, uint8_t* out, crnn_stream_t stream) {
  if (!src || !src_offset || !src_h || !src_w || !out_w || !out) return crnn_fail(CRNN_INVALID_VALUE, "resize_lines_u8: null pointer");
  if (N <= 0 || W < 8 || W % 4) return crnn_fail(CRNN_INVALID_VALUE, "resize_lines_u8: bad shape N = %d, W = %d (W a multiple of 4, >= 8)", N, W);
  if (max_h < 1 || max_h > RS_MAX_H)
    return crnn_fail(CRNN_INVALID_VALUE, "resize_lines_u8: max_h = %d outside [1, %d]", max_h, RS_MAX_H);
  if (reinterpret_cast<uintptr_t>(out) & 3) return crnn_fail(CRNN_INVALID_VALUE, "resize_lines_u8: out must be 4-byte aligned");
  if ((W + RS_TILE - 1) / RS_TILE > 65535)
    return crnn_fail(CRNN_UNSUPPORTED, "resize_lines_u8: W = %d is beyond the kernel (<= %d)", W, 65535 * RS_TILE);
  return resize_lines_u8_launch(src, src_offset, src_h, src_w, out_w, N, W, max_h, out, reinterpret_cast<cudaStream_t>(stream));
}
