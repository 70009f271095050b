// HBM-bound / SIMT kernels of the forward path: BatchNorm finalize/apply, weight re-layout (f32 TF layouts -> bf16 K-major GEMM
// operands), L2 term, loss reduce.
#include "kernels.cuh"

namespace {

// ------------------------------------------------------------------------------------------------
// BatchNorm with batch statistics (tf.contrib.layers.batch_norm(is_training=True), network.py:177-178)
// ------------------------------------------------------------------------------------------------
__global__ void bn_finalize_kernel(const double* __restrict__ stats, double count, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float eps, float* __restrict__ scale,
                                   float* __restrict__ shift, float* __restrict__ save_mean,
                                   float* __restrict__ save_invstd, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double mean = stats[c] / count;
  double var = stats[C + c] / count - mean * mean;      // population variance
  if (var < 0) var = 0;
  const double invstd = 1.0 / sqrt(var + (double)eps);
  const float sc = (float)(gamma[c] * invstd);
  scale[c] = sc;
  shift[c] = (float)(beta[c] - mean * gamma[c] * invstd);
  save_mean[c] = (float)mean;
  save_invstd[c] = (float)invstd;
}

__device__ __forceinline__ uint32_t bn_relu2(uint32_t v, float s0, float h0, float s1, float h1) {
  return ptx::pack_bf16x2(fmaxf(fmaf(ptx::bf16_lo(v), s0, h0), 0.f), fmaxf(fmaf(ptx::bf16_hi(v), s1, h1), 0.f));
}

// in/out [rows, C] bf16, 8 channels per thread
__global__ void __launch_bounds__(256) bn_apply_relu_kernel(const uint4* __restrict__ in, uint4* __restrict__ out,
                                                            const float* __restrict__ scale,
                                                            const float* __restrict__ shift, size_t nvec, int C) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nvec) return;
  const int c = (int)((i * 8) % C);
  const float4 s0 = __ldg(reinterpret_cast<const float4*>(scale + c)), s1 = __ldg(reinterpret_cast<const float4*>(scale + c + 4));
  const float4 h0 = __ldg(reinterpret_cast<const float4*>(shift + c)), h1 = __ldg(reinterpret_cast<const float4*>(shift + c + 4));
  uint4 v = __ldg(in + i);
  v.x = bn_relu2(v.x, s0.x, h0.x, s0.y, h0.y);
  v.y = bn_relu2(v.y, s0.z, h0.z, s0.w, h0.w);
  v.z = bn_relu2(v.z, s1.x, h1.x, s1.y, h1.y);
  v.w = bn_relu2(v.w, s1.z, h1.z, s1.w, h1.w);
  out[i] = v;
}

// in [P, 2*Wo, C] -> out [P, Wo, C]: BN + ReLU then max over adjacent pairs of the Wd axis (pool3, LSTM_train.py:33)
__global__ void __launch_bounds__(256) bn_apply_relu_pool12_kernel(const uint4* __restrict__ in, uint4* __restrict__ out,
                                                                   const float* __restrict__ scale,
                                                                   const float* __restrict__ shift, size_t nvec_out,
                                                                   int C) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nvec_out) return;
  const int vpc = C / 8;                                 // vectors per position
  const size_t pos = i / vpc;
  const int cv = (int)(i - pos * vpc);
  const int c = cv * 8;
  const float4 s0 = __ldg(reinterpret_cast<const float4*>(scale + c)), s1 = __ldg(reinterpret_cast<const float4*>(scale + c + 4));
  const float4 h0 = __ldg(reinterpret_cast<const float4*>(shift + c)), h1 = __ldg(reinterpret_cast<const float4*>(shift + c + 4));
  uint4 a = __ldg(in + (2 * pos) * vpc + cv), b = __ldg(in + (2 * pos + 1) * vpc + cv);
  uint4 o;
  o.x = ptx::hmax2_bf16(bn_relu2(a.x, s0.x, h0.x, s0.y, h0.y), bn_relu2(b.x, s0.x, h0.x, s0.y, h0.y));
  o.y = ptx::hmax2_bf16(bn_relu2(a.y, s0.z, h0.z, s0.w, h0.w), bn_relu2(b.y, s0.z, h0.z, s0.w, h0.w));
  o.z = ptx::hmax2_bf16(bn_relu2(a.z, s1.x, h1.x, s1.y, h1.y), bn_relu2(b.z, s1.x, h1.x, s1.y, h1.y));
  o.w = ptx::hmax2_bf16(bn_relu2(a.w, s1.z, h1.z, s1.w, h1.w), bn_relu2(b.w, s1.z, h1.z, s1.w, h1.w));
  out[i] = o;
}

// ---- per-line BatchNorm of packed evaluation (crnn_forward_lines): every line normalises over its own W_i positions, as when it
// is evaluated alone.  line_w [N] = clamped line widths; a line's positions are its H rows h < line_w / 4 times Wd.
// stats [N][2][C] -> bn [N][4][C] (scale, shift, mean, invstd); one thread per (line, channel), count = line_w[n] (= H2_i * 4)
__global__ void bn_finalize_lines_kernel(const double* __restrict__ stats, const int* __restrict__ line_w, const float* __restrict__ gamma,
                                         const float* __restrict__ beta, float eps, float* __restrict__ bn, int N, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  const int n = i / C, c = i - n * C;
  const double count = (double)line_w[n];
  const double* st = stats + (size_t)n * 2 * C;
  float* o = bn + (size_t)n * 4 * C;
  const double mean = st[c] / count;
  double var = st[C + c] / count - mean * mean;        // population variance
  if (var < 0) var = 0;
  const double invstd = 1.0 / sqrt(var + (double)eps);
  o[c] = (float)(gamma[c] * invstd);
  o[C + c] = (float)(beta[c] - mean * gamma[c] * invstd);
  o[2 * C + c] = (float)mean;
  o[3 * C + c] = (float)invstd;
}

// bn_apply_relu_kernel with each line's own scale / shift; positions at h >= line_w / 4 are written as zero (SAME padding of the
// next conv).  in/out [N, H, Wd, C]
__global__ void __launch_bounds__(256) bn_apply_relu_lines_kernel(const uint4* __restrict__ in, uint4* __restrict__ out,
                                                                  const float* __restrict__ bn, const int* __restrict__ line_w,
                                                                  size_t nvec, int H, int Wd, int C) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nvec) return;
  const int vpc = C / 8;
  const size_t pos = i / vpc;
  const int c = (int)(i - pos * vpc) * 8;
  const size_t row = pos / Wd;                           // n * H + h
  const int n = (int)(row / H), h = (int)(row - (size_t)n * H);
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (h < (__ldg(line_w + n) >> 2)) {
    const float* scale = bn + (size_t)n * 4 * C;
    const float* shift = scale + C;
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(scale + c)), s1 = __ldg(reinterpret_cast<const float4*>(scale + c + 4));
    const float4 h0 = __ldg(reinterpret_cast<const float4*>(shift + c)), h1 = __ldg(reinterpret_cast<const float4*>(shift + c + 4));
    v = __ldg(in + i);
    v.x = bn_relu2(v.x, s0.x, h0.x, s0.y, h0.y);
    v.y = bn_relu2(v.y, s0.z, h0.z, s0.w, h0.w);
    v.z = bn_relu2(v.z, s1.x, h1.x, s1.y, h1.y);
    v.w = bn_relu2(v.w, s1.z, h1.z, s1.w, h1.w);
  }
  out[i] = v;
}

// bn_apply_relu_pool12_kernel with each line's own scale / shift and zero at h >= line_w / 4.  in [N, H, 2*Wo, C] -> out [N, H, Wo, C]
__global__ void __launch_bounds__(256) bn_apply_relu_pool12_lines_kernel(const uint4* __restrict__ in, uint4* __restrict__ out,
                                                                         const float* __restrict__ bn, const int* __restrict__ line_w,
                                                                         size_t nvec_out, int H, int Wo, int C) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nvec_out) return;
  const int vpc = C / 8;
  const size_t pos = i / vpc;
  const int cv = (int)(i - pos * vpc);
  const int c = cv * 8;
  const size_t row = pos / Wo;
  const int n = (int)(row / H), h = (int)(row - (size_t)n * H);
  uint4 o = make_uint4(0u, 0u, 0u, 0u);
  if (h < (__ldg(line_w + n) >> 2)) {
    const float* scale = bn + (size_t)n * 4 * C;
    const float* shift = scale + C;
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(scale + c)), s1 = __ldg(reinterpret_cast<const float4*>(scale + c + 4));
    const float4 h0 = __ldg(reinterpret_cast<const float4*>(shift + c)), h1 = __ldg(reinterpret_cast<const float4*>(shift + c + 4));
    const uint4 a = __ldg(in + (2 * pos) * vpc + cv), b = __ldg(in + (2 * pos + 1) * vpc + cv);
    o.x = ptx::hmax2_bf16(bn_relu2(a.x, s0.x, h0.x, s0.y, h0.y), bn_relu2(b.x, s0.x, h0.x, s0.y, h0.y));
    o.y = ptx::hmax2_bf16(bn_relu2(a.y, s0.z, h0.z, s0.w, h0.w), bn_relu2(b.y, s0.z, h0.z, s0.w, h0.w));
    o.z = ptx::hmax2_bf16(bn_relu2(a.z, s1.x, h1.x, s1.y, h1.y), bn_relu2(b.z, s1.x, h1.x, s1.y, h1.y));
    o.w = ptx::hmax2_bf16(bn_relu2(a.w, s1.z, h1.z, s1.w, h1.w), bn_relu2(b.w, s1.z, h1.z, s1.w, h1.w));
  }
  out[i] = o;
}

// ---- moving statistics (tf.contrib.layers.batch_norm's moving_mean / moving_variance, non-fused, zero_debias = False).
// Every operation is an explicitly rounded f64 operation (no fma contraction), so an fp64 restatement predicts every bit.
// One thread per (layer, channel): stats [2 layers][sum, sum of squares][512] of the training forward, count = positions of the
// (global) batch; moving [2 layers][mean, variance][512] f32 in place:  moving -= (moving - batch value) * (1 - decay)
__global__ void bn_moving_update_kernel(const double* __restrict__ stats, double count, float* __restrict__ moving, float decay) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * 512) return;
  const int l = i >> 9, c = i & 511;
  const double* st = stats + l * 1024;
  const double mean = __ddiv_rn(st[c], count);
  double var = __dsub_rn(__ddiv_rn(st[512 + c], count), __dmul_rn(mean, mean));    // population variance, as the forward's
  if (var < 0) var = 0;
  const double f = __dsub_rn(1.0, (double)decay);
  float* mv = moving + l * 1024;
  const double m0 = mv[c], v0 = mv[512 + c];
  mv[c] = (float)__dsub_rn(m0, __dmul_rn(__dsub_rn(m0, mean), f));
  mv[512 + c] = (float)__dsub_rn(v0, __dmul_rn(__dsub_rn(v0, var), f));
}

// Fold the moving statistics of one BN layer into its conv: s = gamma / sqrt(var + eps) (f64), B'[co][k] = bf16(W[k][co] * s) (one
// rounding), b'[co] = f32((b - mean) * s + beta) (one rounding); scale_out keeps s for the fp8 column scales.  One CTA per channel.
__global__ void __launch_bounds__(256) bn_fold_kernel(const float* __restrict__ w, int K, int Cout, const float* __restrict__ bias,
                                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                                      const float* __restrict__ moving, float eps, __nv_bfloat16* __restrict__ bout,
                                                      float* __restrict__ bias_out, double* __restrict__ scale_out) {
  const int co = blockIdx.x;
  const double s = __ddiv_rn((double)gamma[co], __dsqrt_rn(__dadd_rn((double)moving[Cout + co], (double)eps)));
  for (int r = threadIdx.x; r < K; r += 256) bout[(size_t)co * K + r] = __double2bfloat16(__dmul_rn((double)__ldg(w + (size_t)r * Cout + co), s));
  if (threadIdx.x == 0) {
    bias_out[co] = (float)__dadd_rn(__dmul_rn(__dsub_rn((double)bias[co], (double)moving[co]), s), (double)beta[co]);
    scale_out[co] = s;
  }
}

// line widths as every packed-evaluation kernel reads them: clamped to [8, W] and rounded down to a multiple of 4
__global__ void clamp_line_width_kernel(const int* __restrict__ in, int* __restrict__ out, int N, int W) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) out[i] = min(max(in[i], 8), W) & ~3;
}

// ------------------------------------------------------------------------------------------------
// weight re-layout: dst[perm(c)][r] (bf16, K-major GEMM B operand) = src[r][c] (f32, TF layout)
// perm_mode 0: identity; upc > 0 (= LSTM_GATE_UNITS): LSTM gate permutation  j = g*256+u  ->  (u/upc)*4*upc + g*upc + u%upc
// (a tile of 4*upc consecutive rows then holds [i|j|f|o] of upc hidden units)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int lstm_perm(int j, int upc) {
  const int g = j >> 8, u = j & 255;
  return (u / upc) * 4 * upc + g * upc + (u % upc);
}
__global__ void __launch_bounds__(256) transpose_cast_kernel(const float* __restrict__ src, int R, int Cc, int ld_src,
                                                             __nv_bfloat16* __restrict__ dst, int ld_dst,
                                                             int perm_mode) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    const int r = r0 + i, c = c0 + tx;
    tile[i][tx] = (r < R && c < Cc) ? __ldg(src + (size_t)r * ld_src + c) : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, r = r0 + tx;
    if (c < Cc && r < R) {
      const int dc = perm_mode ? lstm_perm(c, perm_mode) : c;
      dst[(size_t)dc * ld_dst + r] = __float2bfloat16_rn(tile[tx][i]);
    }
  }
}
__global__ void lstm_bias_prep_kernel(const float* __restrict__ b_fw, const float* __restrict__ b_bw,
                                      float* __restrict__ xbias, int upc) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;   // 0..2047
  if (j >= 2048) return;
  const int dir = j >> 10, jj = j & 1023;
  const float v = (dir ? b_bw : b_fw)[jj] + (((jj >> 8) == 2) ? 1.0f : 0.0f);   // forget_bias = 1.0 on gate f
  xbias[dir * 1024 + lstm_perm(jj, upc)] = v;
}

// ------------------------------------------------------------------------------------------------
// L2 term and total loss (network.py:630-637,655,660-662)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ params, SumsqSegs segs,
                                                    double* __restrict__ out) {
  double acc = 0.0;
  for (int sgi = 0; sgi < segs.n; ++sgi) {
    const float4* p = reinterpret_cast<const float4*>(params + segs.off[sgi]);
    const size_t nv = segs.cnt[sgi] / 4;
    float part = 0.f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (size_t)gridDim.x * blockDim.x) {
      const float4 v = __ldg(p + i);
      part += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    acc += part;
  }
  __shared__ double red[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int i = 0; i < 8; ++i) t += red[i];
    atomicAdd(out, t);
  }
}

__global__ void __launch_bounds__(256) total_loss_kernel(const float* __restrict__ costs, int N,
                                                         const double* __restrict__ sumsq, float wd,
                                                         float* __restrict__ loss) {
  double acc = 0.0;
  for (int i = threadIdx.x; i < N; i += 256) acc += costs[i];
  __shared__ double red[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int i = 0; i < 8; ++i) t += red[i];
    *loss = (float)(t / N + (wd > 0.f ? 0.5 * (double)wd * (*sumsq) : 0.0));
  }
}

__global__ void bf16_to_f32_kernel(const __nv_bfloat16* __restrict__ in, float* __restrict__ out, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __bfloat162float(in[i]);
}

}  // namespace

// ------------------------------------------------------------------------------------------------ launchers
int launch_bn_finalize(const double* stats, double count, const float* gamma, const float* beta, float eps, float* scale,
                       float* shift, float* save_mean, float* save_invstd, int C, cudaStream_t st) {
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(stats, count, gamma, beta, eps, scale, shift, save_mean, save_invstd, C);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
int launch_bn_apply_relu(const __nv_bfloat16* in, __nv_bfloat16* out, const float* scale, const float* shift, size_t rows,
                         int C, cudaStream_t st) {
  const size_t nvec = rows * C / 8;
  bn_apply_relu_kernel<<<(unsigned)((nvec + 255) / 256), 256, 0, st>>>(reinterpret_cast<const uint4*>(in),
                                                                       reinterpret_cast<uint4*>(out), scale, shift, nvec, C);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
int launch_bn_apply_relu_pool12(const __nv_bfloat16* in, __nv_bfloat16* out, const float* scale, const float* shift,
                                size_t out_positions, int C, cudaStream_t st) {
  const size_t nvec = out_positions * C / 8;
  bn_apply_relu_pool12_kernel<<<(unsigned)((nvec + 255) / 256), 256, 0, st>>>(
      reinterpret_cast<const uint4*>(in), reinterpret_cast<uint4*>(out), scale, shift, nvec, C);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
int launch_bn_moving_update(const double* stats, double count, float* moving, float decay, cudaStream_t st) {
  bn_moving_update_kernel<<<4, 256, 0, st>>>(stats, count, moving, decay);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
int launch_bn_fold(const float* w, int K, int Cout, const float* bias, const float* gamma, const float* beta, const float* moving, float eps,
                   __nv_bfloat16* bout, float* bias_out, double* scale_out, cudaStream_t st) {
  bn_fold_kernel<<<Cout, 256, 0, st>>>(w, K, Cout, bias, gamma, beta, moving, eps, bout, bias_out, scale_out);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
int launch_clamp_line_width(const int* in, int* out, int N, int W, cudaStream_t st) {
  clamp_line_width_kernel<<<(N + 255) / 256, 256, 0, st>>>(in, out, N, W);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
int launch_bn_finalize_lines(const double* stats, const int* line_w, const float* gamma, const float* beta, float eps, float* bn, int N,
                             int C, cudaStream_t st) {
  bn_finalize_lines_kernel<<<(N * C + 127) / 128, 128, 0, st>>>(stats, line_w, gamma, beta, eps, bn, N, C);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
int launch_bn_apply_relu_lines(const __nv_bfloat16* in, __nv_bfloat16* out, const float* bn, const int* line_w, int N, int H, int Wd,
                               int C, cudaStream_t st) {
  const size_t nvec = (size_t)N * H * Wd * C / 8;
  bn_apply_relu_lines_kernel<<<(unsigned)((nvec + 255) / 256), 256, 0, st>>>(reinterpret_cast<const uint4*>(in), reinterpret_cast<uint4*>(out),
                                                                             bn, line_w, nvec, H, Wd, C);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
int launch_bn_apply_relu_pool12_lines(const __nv_bfloat16* in, __nv_bfloat16* out, const float* bn, const int* line_w, int N, int H,
                                      int Wo, int C, cudaStream_t st) {
  const size_t nvec = (size_t)N * H * Wo * C / 8;
  bn_apply_relu_pool12_lines_kernel<<<(unsigned)((nvec + 255) / 256), 256, 0, st>>>(
      reinterpret_cast<const uint4*>(in), reinterpret_cast<uint4*>(out), bn, line_w, nvec, H, Wo, C);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
int launch_transpose_cast(const float* src, int R, int Cc, int ld_src, __nv_bfloat16* dst, int ld_dst, bool lstm_gates,
                          cudaStream_t st) {
  dim3 grid((Cc + 31) / 32, (R + 31) / 32);
  transpose_cast_kernel<<<grid, 256, 0, st>>>(src, R, Cc, ld_src, dst, ld_dst, lstm_gates ? LSTM_GATE_UNITS : 0);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
int launch_lstm_bias_prep(const float* b_fw, const float* b_bw, float* xbias, cudaStream_t st) {
  lstm_bias_prep_kernel<<<8, 256, 0, st>>>(b_fw, b_bw, xbias, LSTM_GATE_UNITS);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
int launch_sumsq(const float* params, const SumsqSegs& segs, double* out, cudaStream_t st) {
  CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(double), st));
  sumsq_kernel<<<296, 256, 0, st>>>(params, segs, out);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
int launch_total_loss(const float* costs, int N, const double* sumsq, float wd, float* loss, cudaStream_t st) {
  total_loss_kernel<<<1, 256, 0, st>>>(costs, N, sumsq, wd, loss);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
int launch_bf16_to_f32(const __nv_bfloat16* in, float* out, size_t n, cudaStream_t st) {
  bf16_to_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, out, n);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
