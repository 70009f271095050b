// Launchers for the SIMT / HBM-bound kernels (kernels.cu).
#pragma once
#include "common.cuh"

struct SumsqSegs {
  int n;
  long long off[8];
  long long cnt[8];
};

int launch_bn_finalize(const double* stats, double count, const float* gamma, const float* beta, float eps, float* scale,
                       float* shift, float* save_mean, float* save_invstd, int C, cudaStream_t st);
int launch_bn_apply_relu(const __nv_bfloat16* in, __nv_bfloat16* out, const float* scale, const float* shift, size_t rows,
                         int C, cudaStream_t st);
int launch_bn_apply_relu_pool12(const __nv_bfloat16* in, __nv_bfloat16* out, const float* scale, const float* shift,
                                size_t out_positions, int C, cudaStream_t st);
// packed evaluation (crnn_forward_lines): line widths clamped once, per-line BatchNorm finalize (bn [N][4][C] from stats [N][2][C])
// and apply (zero at h >= line_w / 4)
int launch_clamp_line_width(const int* in, int* out, int N, int W, cudaStream_t st);
int launch_bn_finalize_lines(const double* stats, const int* line_w, const float* gamma, const float* beta, float eps, float* bn, int N,
                             int C, cudaStream_t st);
int launch_bn_apply_relu_lines(const __nv_bfloat16* in, __nv_bfloat16* out, const float* bn, const int* line_w, int N, int H, int Wd,
                               int C, cudaStream_t st);
int launch_bn_apply_relu_pool12_lines(const __nv_bfloat16* in, __nv_bfloat16* out, const float* bn, const int* line_w, int N, int H,
                                      int Wo, int C, cudaStream_t st);
// moving BatchNorm statistics of conv4_1 / conv4_2: the per-step update from the training forward's f64 sums, and the fold of one
// layer's statistics into its conv (bf16 B operand [Cout][K], f32 bias, f64 per-channel scale)
int launch_bn_moving_update(const double* stats, double count, float* moving, float decay, cudaStream_t st);
int launch_bn_fold(const float* w, int K, int Cout, const float* bias, const float* gamma, const float* beta, const float* moving, float eps,
                   __nv_bfloat16* bout, float* bias_out, double* scale_out, cudaStream_t st);
// lstm_gates: the columns are LSTM gate columns, stored permuted (LSTM_GATE_UNITS units per [i|j|f|o] tile)
int launch_transpose_cast(const float* src, int R, int Cc, int ld_src, __nv_bfloat16* dst, int ld_dst, bool lstm_gates,
                          cudaStream_t st);
int launch_lstm_bias_prep(const float* b_fw, const float* b_bw, float* xbias, cudaStream_t st);
int launch_sumsq(const float* params, const SumsqSegs& segs, double* out, cudaStream_t st);
int launch_total_loss(const float* costs, int N, const double* sumsq, float wd, float* loss, cudaStream_t st);
int launch_bf16_to_f32(const __nv_bfloat16* in, float* out, size_t n, cudaStream_t st);
