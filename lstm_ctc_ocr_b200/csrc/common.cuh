// Shared host/device helpers for libcrnnctc.so.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/crnn_ctc.h"
#include "ptx.cuh"

int crnn_fail(int status, const char* fmt, ...);   // records crnn_last_error(), returns status

#define CUDA_TRY(expr)                                                                             \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      return crnn_fail(CRNN_CUDA_ERROR, "%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
  } while (0)

#define CRNN_TRY(expr)            \
  do {                            \
    int _s = (expr);              \
    if (_s != CRNN_OK) return _s; \
  } while (0)

// A caller's pointer that the kernels access in units wider than its element type (f32 rows as float4, uint8 pixels as 4-byte
// words) must be `align`-byte aligned; a misaligned one would fault on the device and poison the caller's CUDA context, so the
// entry points refuse it on the host before anything is enqueued.  A null pointer passes (the null checks are the callers').
inline int check_aligned(const void* p, unsigned align, const char* fn, const char* arg) {
  if ((reinterpret_cast<uintptr_t>(p) & (align - 1)) != 0)
    return crnn_fail(CRNN_INVALID_VALUE, "%s: %s must be %u-byte aligned", fn, arg, align);
  return CRNN_OK;
}

// ---- input pixels: the f32 data tensor [N, W, 32] or its uint8 twin (the crnn_*_u8 entry points).  A byte u is the pixel
// x = (float)u / 255.0f, an IEEE round-to-nearest division (numpy's u.astype(float32) / float32(255)): the value the f32 feed
// holds, so both feeds give conv1 the same operands.  A reciprocal multiply alone differs from that quotient on 126 of the 256
// bytes; one FMA correction of it (q0 = u * r, q = q0 + (u - q0 * 255) * r, r = f32(1/255)) is the quotient on all 256 (checked
// exhaustively in exact arithmetic by tests/test_u8_feed_cpu.py) at a third of the instructions of the division.
// Pixels4<T> loads 4 consecutive pixels of a row (16 bytes of f32, one 4-byte word of u8) and widens them where they are used.
__device__ __forceinline__ float u8_pixel(uint32_t u) {
  constexpr float r = 1.0f / 255.0f;
  const float x = (float)u;
  const float q0 = __fmul_rn(x, r);
  return __fmaf_rn(__fmaf_rn(-q0, 255.0f, x), r, q0);
}
template <typename T> struct Pixels4;
template <> struct Pixels4<float> {
  using Raw = float4;
  static __device__ __forceinline__ Raw zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
  static __device__ __forceinline__ Raw load(const float* row, int c4) { return __ldg(reinterpret_cast<const float4*>(row) + c4); }
  static __device__ __forceinline__ float4 f32(const Raw& v) { return v; }
};
template <> struct Pixels4<uint8_t> {
  using Raw = uint32_t;
  static __device__ __forceinline__ Raw zero() { return 0u; }
  static __device__ __forceinline__ Raw load(const uint8_t* row, int c4) { return __ldg(reinterpret_cast<const unsigned int*>(row) + c4); }
  static __device__ __forceinline__ float4 f32(const Raw& v) {
    return make_float4(u8_pixel(v & 255u), u8_pixel((v >> 8) & 255u), u8_pixel((v >> 16) & 255u), u8_pixel(v >> 24));
  }
};
__device__ __forceinline__ float pixel_f32(float x) { return x; }
__device__ __forceinline__ float pixel_f32(uint8_t u) { return u8_pixel(u); }

// hidden units per [i|j|f|o] gate tile of the permuted LSTM weight columns: one CTA of the 8-CTA recurrence clusters owns 32
// units (lstm.cuh), so gate column j = g*256 + u sits at (u/32)*128 + g*32 + u%32
constexpr int LSTM_GATE_UNITS = 32;

// ---- saved LSTM state (training): written by the forward recurrence kernels, read by the BPTT kernels.  Both access it with
// lane = sample row of a 128-row batch tile, so the layout keeps the 128 rows of a tile adjacent: a warp's 32 lanes store / load
// 32 consecutive 16-byte vectors (one 512-byte segment) instead of 32 sectors that are T*2 KB apart.
//   gates [dir*tiles + tile][step][gate i,j,f,o][unit/8 = 32 chunks][row 128][8 bf16]      (post-activation gate values)
//   csave [dir*tiles + tile][step][unit/4 = 64 chunks][row 128][4 f32]                      (cell state after the step)
constexpr size_t LSTM_GCHUNK_STRIDE = 128 * 8;                 // elements between unit chunks of 8
constexpr size_t LSTM_GATE_STRIDE = 32 * LSTM_GCHUNK_STRIDE;   // elements between gates
constexpr size_t LSTM_GSTEP_STRIDE = 4 * LSTM_GATE_STRIDE;     // elements between steps
constexpr size_t LSTM_CCHUNK_STRIDE = 128 * 4;                 // elements between unit chunks of 4
constexpr size_t LSTM_CSTEP_STRIDE = 64 * LSTM_CCHUNK_STRIDE;  // elements between steps
// dts = (dir*tiles_per_dir + tile) * T + step; `unit` must be a multiple of 8 (gates) / 4 (csave)
__host__ __device__ __forceinline__ size_t lstm_gate_off(size_t dts, int g, int unit, int row) {
  return dts * LSTM_GSTEP_STRIDE + (size_t)g * LSTM_GATE_STRIDE + (size_t)(unit >> 3) * LSTM_GCHUNK_STRIDE + (size_t)row * 8;
}
__host__ __device__ __forceinline__ size_t lstm_c_off(size_t dts, int unit, int row) {
  return dts * LSTM_CSTEP_STRIDE + (size_t)(unit >> 2) * LSTM_CCHUNK_STRIDE + (size_t)row * 4;
}
