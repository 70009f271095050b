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
