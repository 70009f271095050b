// Internal launcher of resize.cu's Pillow BILINEAR resize, shared by crnn_resize_lines_u8 and the device line renderer
// (render.cu), so the library holds one resampling implementation.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// The launch behind crnn_resize_lines_u8, without its argument checks: the caller guarantees N >= 1, W >= 8 and a multiple of 4,
// 1 <= max_h <= 1024, a 4-byte aligned `out` and W <= 65535 * 32.  Returns CRNN_OK or CRNN_CUDA_ERROR (crnn_last_error() set).
int resize_lines_u8_launch(const uint8_t* src, const int64_t* src_offset, const int* src_h, const int* src_w, const int* out_w,
                           int N, int W, int max_h, uint8_t* out, cudaStream_t stream);
