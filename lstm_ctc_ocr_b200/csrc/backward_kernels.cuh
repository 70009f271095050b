// Launchers for the non-GEMM backward / optimizer kernels (backward_kernels.cu).
#pragma once
#include "common.cuh"

struct WdSegs {
  int n;
  long long off[8];
  long long cnt[8];
};

int launch_dlogits_rows(const float* dlogits, __nv_bfloat16* rows, float* dbias, int T, int N, int H, cudaStream_t st);
// lstm_gates: the columns are the permuted gate columns of both LSTM directions (2 x 1024), summed into TF order `dir_stride` apart
int launch_colsum_bf16(const __nv_bfloat16* src, long long R, int C, float* out, bool lstm_gates, long long dir_stride, cudaStream_t st);
int launch_colsum_masked_bf16(const __nv_bfloat16* src, const __nv_bfloat16* mask, long long R, int C, float* out, cudaStream_t st);
// conv4_2's BatchNorm + ReLU + pool3 backward sums (dout pooled: out_positions = pooled positions)
int launch_bn_bwd_reduce(const __nv_bfloat16* dout, const __nv_bfloat16* x_pre, const float* bn, double* sums, size_t out_positions, int C,
                         cudaStream_t st);
int launch_bn_bwd_apply(bool pool, const __nv_bfloat16* dout, const __nv_bfloat16* x_pre, __nv_bfloat16* dx, const float* bn,
                        const float* gamma, const double* sums, const double* sums_local, double count, size_t out_positions, int C,
                        float* coef, float* dgamma, float* dbeta, cudaStream_t st);
int launch_unpool_relu_bwd(int win, const __nv_bfloat16* dpool, const __nv_bfloat16* pooled, const uint8_t* argmax,
                           __nv_bfloat16* dpre, size_t out_positions, int Hp, int Wp, int C, cudaStream_t st);
int launch_dgrad_weight(const float* w, __nv_bfloat16* bd, int Cin, int Cout, cudaStream_t st);
int launch_conv5_dgrad_weight(const float* w, __nv_bfloat16* bd, cudaStream_t st);
int launch_lstm_bwd_weight(const float* w_fw, const float* w_bw, __nv_bfloat16* bxb, __nv_bfloat16* bhb, cudaStream_t st);
int launch_cast_bf16(const float* src, __nv_bfloat16* dst, size_t n, cudaStream_t st);
int launch_grad_finish(float* grads, const float* params, const WdSegs& segs, float wd, long long total, double* sumsq, cudaStream_t st);
int launch_clip_adam(float* params, const float* grads, float* m, float* v, const double* sumsq, float grad_mul, float clip, float lr_t,
                     float b1, float b2, float eps, long long total, cudaStream_t st);
int launch_clip_momentum(float* params, const float* grads, float* accum, const double* sumsq, float grad_mul, float clip, float lr,
                         float momentum, long long total, cudaStream_t st);
int launch_clip_rmsprop(float* params, const float* grads, float* mom, float* ms, const double* sumsq, float grad_mul, float clip,
                        float lr, float decay, float momentum, float eps, long long total, cudaStream_t st);
