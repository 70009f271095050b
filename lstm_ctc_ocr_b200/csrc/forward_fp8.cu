// FP8 inference path (crnn_config.compute_dtype = 4): conv3_1, conv3_2, conv4_1, conv4_2 and conv5 -- 2 921 of the 3 240 conv
// GFLOP at batch 1024 x 32x256 -- run on e4m3 wgmma operands (gemm::gemm_kernel<..., KIND = 2>, twice the bf16 tensor rate on
// H100); everything else is the bf16 path of model.cu unchanged.  Forward only.
//
// Scales (fixed, so that every stage can be restated exactly):
//   weights      s_w[co] = amax_co(|w|) / 448 (f32 division; 1 when the amax is 0), B[co][k] = e4m3(w[k][co] / s_w[co])
//                (round to nearest even, saturating), K-major [Cout][K] in the natural (kh, kw, ci) order; prepared when the
//                parameters change, like the bf16 copies.
//   activations  one static power-of-two scale per fp8 operand -- a2, a3, a3p, a4a, a4b (the A operands of the five GEMMs):
//                s = 2^max(-126, ceil(log2(amax / 448))) over the f32 quotient, 1 when the amax is 0 or not finite.  Dividing by
//                a power of two is exact, so the producers store e4m3(y / s) and the consumers' epilogues undo it exactly;
//                values above the calibrated range saturate to +-448.
//   epilogues    y = acc * colscale[co] + bias[co] (one fma), colscale = s_in * s_w (exact: s_in is a power of two); then
//                ReLU / pooling as on the bf16 path, and e4m3(y / s_out) where the next consumer is fp8.
// Producers write e4m3 themselves: conv2_swap_kernel<false, LINES, true> (a2), frag_epilogue EPI_RELU / EPI_RELU_POOL12 with
// KIND 2 (a3, a3p), bn_apply_e4m3_kernel (a4a, a4b).  conv4_x keep their bf16 pre-BN output and f64 batch statistics, conv5
// its bf16 output.  With moving BatchNorm statistics (crnn_model_set_bn_statistics) the BN folds into conv4_x's colscale and bias,
// and their EPI_RELU / EPI_RELU_POOL12 epilogues write e4m3 a4a / a4b themselves.
// Calibration (crnn_model_calibrate_fp8) runs the bf16 front end on a caller-supplied batch and reduces the five amaxes on the
// device (atomicMax on the f32 bits of non-negative values: deterministic); the scales never leave the device.
#include <cmath>
#include <cstring>
#include <string>

#include "conv_swap.cuh"
#include "gemm_launch.h"
#include "kernels.cuh"
#include "model_internal.h"

namespace fp8 {

constexpr int kLayers = 5;
struct LayerSpec { const char* name; int K, Cout, Cin; };
static const LayerSpec kL[kLayers] = {{"conv3_1", 1152, 256, 128}, {"conv3_2", 2304, 256, 256}, {"conv4_1", 2304, 512, 256},
                                      {"conv4_2", 4608, 512, 512}, {"conv5", 2048, 512, 1024}};

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// one CTA per output channel: s_w[co] = amax / 448, dst[co][r] = e4m3(src[r][co] / s_w[co])
__global__ void __launch_bounds__(256) weight_quant_kernel(const float* __restrict__ src, int K, int Cout, uint8_t* __restrict__ dst,
                                                           float* __restrict__ wscale) {
  const int co = blockIdx.x;
  float amax = 0.f;
  for (int r = threadIdx.x; r < K; r += 256) amax = fmaxf(amax, fabsf(__ldg(src + (size_t)r * Cout + co)));
  __shared__ float red[8];
  __shared__ float s_sh;
  amax = warp_max(amax);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = red[0];
    for (int i = 1; i < 8; ++i) a = fmaxf(a, red[i]);
    const float s = a > 0.f ? __fdiv_rn(a, 448.f) : 1.f;
    s_sh = s;
    wscale[co] = s;
  }
  __syncthreads();
  const float s = s_sh;
  for (int r = threadIdx.x; r < K; r += 256)
    dst[(size_t)co * K + r] = (uint8_t)(ptx::pack_e4m3x2(__fdiv_rn(__ldg(src + (size_t)r * Cout + co), s), 0.f) & 0xFFu);
}

// amax of a bf16 tensor (8 values per thread and step) -> atomicMax on the f32 bits (|x| >= 0 orders like its bits)
__global__ void __launch_bounds__(256) amax_bf16_kernel(const uint4* __restrict__ in, size_t nvec, unsigned* __restrict__ out) {
  float m = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    const uint4 v = __ldg(in + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) m = fmaxf(m, fmaxf(fabsf(ptx::bf16_lo(w[k])), fabsf(ptx::bf16_hi(w[k]))));
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}

__device__ __forceinline__ float pow2_scale(float amax) {
  if (!(amax > 0.f) || !isfinite(amax)) return 1.f;
  int e;
  const float m = frexpf(__fdiv_rn(amax, 448.f), &e);     // quotient = m * 2^e, m in [0.5, 1)
  const int c = (m == 0.5f) ? e - 1 : e;                    // ceil(log2(quotient))
  return ldexpf(1.f, c < -126 ? -126 : c);
}

__global__ void scale_finalize_kernel(const unsigned* __restrict__ amax, float* __restrict__ scales) {
  if (threadIdx.x < kLayers) scales[threadIdx.x] = pow2_scale(__uint_as_float(amax[threadIdx.x]));
}

// moving statistics: colscale_m[l][co] = f32(colscale[2 + l][co] * s[l][co]) (f64 product, one rounding), s = the fold's
// gamma / sqrt(var + eps) of conv4_1 (l = 0) / conv4_2 (l = 1); the e4m3 weights stay as they are
__global__ void colscale_moving_kernel(const float* __restrict__ colscale, const double* __restrict__ s, float* __restrict__ colscale_m) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 2 * 512) colscale_m[i] = (float)__dmul_rn((double)colscale[2 * 512 + i], s[i]);
}

// colscale[l][co] = scales[l] * wscale[l][co]   ([5][512]; conv3_x use 256 columns)
__global__ void colscale_kernel(const float* __restrict__ scales, const float* __restrict__ wscale, float* __restrict__ colscale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < kLayers * 512) colscale[i] = scales[i / 512] * wscale[i];
}

// BatchNorm + ReLU (+ max over Wd pairs) into e4m3: out = e4m3(y / *oscale), y = max(relu(fma(x, scale, shift))) in f32.
// in bf16 [N, H, (POOL ? 2 : 1) * Wo, C] -> out e4m3 [N, H, Wo, C], 8 channels per thread.  LINES: each line's own coefficients
// (bn [N][4][C]) and zero at h >= line_w / 4; otherwise bn = [4][C] of the whole batch.
template <bool POOL, bool LINES>
__global__ void __launch_bounds__(256) bn_apply_e4m3_kernel(const uint4* __restrict__ in, uint2* __restrict__ out, const float* __restrict__ bn,
                                                            const int* __restrict__ line_w, const float* __restrict__ oscale, size_t nvec,
                                                            int H, int Wo, int C) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nvec) return;
  const int vpc = C / 8;
  const size_t pos = i / vpc;
  const int cv = (int)(i - pos * vpc);
  const int c = cv * 8;
  const float* scale = bn;
  if (LINES) {
    const size_t row = pos / Wo;
    const int n = (int)(row / H), h = (int)(row - (size_t)n * H);
    if (h >= (__ldg(line_w + n) >> 2)) { out[i] = make_uint2(0u, 0u); return; }
    scale = bn + (size_t)n * 4 * C;
  }
  const float* shift = scale + C;
  const float4 s0 = __ldg(reinterpret_cast<const float4*>(scale + c)), s1 = __ldg(reinterpret_cast<const float4*>(scale + c + 4));
  const float4 h0 = __ldg(reinterpret_cast<const float4*>(shift + c)), h1 = __ldg(reinterpret_cast<const float4*>(shift + c + 4));
  const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
  const float sh[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
  const uint4 a = __ldg(POOL ? in + (2 * pos) * vpc + cv : in + i);
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
  float y[8];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    y[2 * k] = fmaxf(fmaf(ptx::bf16_lo(aw[k]), sc[2 * k], sh[2 * k]), 0.f);
    y[2 * k + 1] = fmaxf(fmaf(ptx::bf16_hi(aw[k]), sc[2 * k + 1], sh[2 * k + 1]), 0.f);
  }
  if (POOL) {
    const uint4 b = __ldg(in + (2 * pos + 1) * vpc + cv);
    const uint32_t bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      y[2 * k] = fmaxf(y[2 * k], fmaxf(fmaf(ptx::bf16_lo(bw[k]), sc[2 * k], sh[2 * k]), 0.f));
      y[2 * k + 1] = fmaxf(y[2 * k + 1], fmaxf(fmaf(ptx::bf16_hi(bw[k]), sc[2 * k + 1], sh[2 * k + 1]), 0.f));
    }
  }
  const float inv = 1.f / __ldg(oscale);
  out[i] = make_uint2(ptx::pack_e4m3x4(y[0] * inv, y[1] * inv, y[2] * inv, y[3] * inv),
                      ptx::pack_e4m3x4(y[4] * inv, y[5] * inv, y[6] * inv, y[7] * inv));
}

// debug tap: e4m3 bytes * scale -> f32
__global__ void dequant_kernel(const uint8_t* __restrict__ in, const float* __restrict__ scale, float* __restrict__ out, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = ptx::e4m3_to_f32(in[i]) * __ldg(scale);
}

struct State {
  void* block = nullptr;
  uint8_t* Wq[kLayers];
  float* wscale;        // [5][512]
  float* scales;        // [5] activation scales: a2, a3, a3p, a4a, a4b
  float* colscale;      // [5][512]
  float* colscale_m;    // [2][512] conv4_x colscale with the moving statistics folded in
  unsigned* amax;       // [5] calibration scratch
  CUtensorMap tB[kLayers];
  bool dirty = true;            // weights changed since the e4m3 copies were made
  bool colscale_dirty = true;   // weight or activation scales changed since colscale was computed
  bool calibrated = false;      // activation scales valid for the current parameters
  bool colscale_m_dirty = true; // colscale or the moving-statistics fold changed since colscale_m was computed
};

// allocated once, by crnn_model_create of an fp8 model: calibration and the forward allocate nothing
static int create_state(crnn_model* m) {
  {
    State* s = new State();
    size_t tot = 0;
    for (int l = 0; l < kLayers; ++l) tot += align_up((size_t)kL[l].K * kL[l].Cout);
    tot += 4 * align_up(kLayers * 512 * 4) + 1024;
    if (cudaMalloc(&s->block, tot) != cudaSuccess) { delete s; return crnn_fail(CRNN_CUDA_ERROR, "fp8: cudaMalloc"); }
    // cudaMemset is ordered on the legacy stream only: wait for it, or a busy legacy stream lets it land after the first forward
    // or calibration on a non-blocking stream has written this block
    if (cudaMemset(s->block, 0, tot) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) {
      cudaFree(s->block); delete s; return crnn_fail(CRNN_CUDA_ERROR, "fp8: cudaMemset");
    }
    uint8_t* p = reinterpret_cast<uint8_t*>(s->block);
    for (int l = 0; l < kLayers; ++l) { s->Wq[l] = p; p += align_up((size_t)kL[l].K * kL[l].Cout); }
    s->wscale = reinterpret_cast<float*>(p); p += align_up(kLayers * 512 * 4);
    s->colscale = reinterpret_cast<float*>(p); p += align_up(kLayers * 512 * 4);
    s->colscale_m = reinterpret_cast<float*>(p); p += align_up(kLayers * 512 * 4);
    s->scales = reinterpret_cast<float*>(p); s->amax = reinterpret_cast<unsigned*>(p + 64);
    for (int l = 0; l < kLayers; ++l) {
      const int st = make_tmap_2d_u8(&s->tB[l], s->Wq[l], kL[l].Cout, kL[l].K, kL[l].K, 256);
      if (st != CRNN_OK) { cudaFree(s->block); delete s; return st; }
    }
    m->fp8 = s;
  }
  return CRNN_OK;
}

}  // namespace fp8

// ------------------------------------------------------------------------------------------------ hooks of model.cu
using fp8::State;

int fp8_create(crnn_model* m) { return fp8::create_state(m); }

void fp8_destroy(crnn_model* m) {
  State* s = reinterpret_cast<State*>(m->fp8);
  if (!s) return;
  if (s->block) cudaFree(s->block);
  delete s;
  m->fp8 = nullptr;
}

void fp8_params_changed(crnn_model* m) {
  State* s = reinterpret_cast<State*>(m->fp8);
  if (!s) return;
  s->dirty = true;
  s->colscale_dirty = true;
  s->calibrated = false;
}

bool fp8_calibrated(const crnn_model* m) {
  const State* s = reinterpret_cast<const State*>(m->fp8);
  return s && s->calibrated;
}

int fp8_prepare(crnn_model* m, cudaStream_t st) {
  State* s = reinterpret_cast<State*>(m->fp8);
  if (s->dirty) {
    for (int l = 0; l < fp8::kLayers; ++l) {
      const fp8::LayerSpec& L = fp8::kL[l];
      fp8::weight_quant_kernel<<<L.Cout, 256, 0, st>>>(m->P(std::string(L.name) + "/weights"), L.K, L.Cout, s->Wq[l], s->wscale + l * 512);
      CUDA_TRY(cudaGetLastError());
    }
    s->dirty = false;
    s->colscale_dirty = true;
  }
  if (s->colscale_dirty) {
    fp8::colscale_kernel<<<(fp8::kLayers * 512 + 255) / 256, 256, 0, st>>>(s->scales, s->wscale, s->colscale);
    CUDA_TRY(cudaGetLastError());
    s->colscale_dirty = false;
    s->colscale_m_dirty = true;
  }
  return CRNN_OK;
}

// after fp8_prepare and bn_fold_moving (`refolded`: the fold ran again)
int fp8_fold_moving(crnn_model* m, bool refolded, cudaStream_t st) {
  State* s = reinterpret_cast<State*>(m->fp8);
  if (refolded || s->colscale_m_dirty) {
    fp8::colscale_moving_kernel<<<4, 256, 0, st>>>(s->colscale, m->bm_scale, s->colscale_m);
    CUDA_TRY(cudaGetLastError());
    s->colscale_m_dirty = false;
  }
  return CRNN_OK;
}

int fp8_plan_maps(Plan& pl) {
  const int N = pl.N;
  CRNN_TRY(make_tmap_nhwc_u8(&pl.q_c31, pl.a2, N, pl.H2, 8, 128, pl.mg3 ? 16 : 4));
  CRNN_TRY(make_tmap_nhwc_u8(&pl.q_c32, pl.a3, N, pl.H2, 8, 256, pl.mg3 ? 16 : 4));
  CRNN_TRY(make_tmap_nhwc_u8(&pl.q_c41, pl.a3p, N, pl.H2, 4, 256, pl.mg4 ? 32 : 8));
  CRNN_TRY(make_tmap_nhwc_u8(&pl.q_c42, pl.a4a, N, pl.H2, 4, 512, pl.mg4 ? 32 : 8));
  CRNN_TRY(make_tmap_2d_u8(&pl.q_c5, pl.a4b, (uint64_t)N * pl.H2, 1024, 1024, 128));
  CRNN_TRY(make_tmap_nhwc_u8(&pl.qO_c2s, pl.a2, N, pl.H2, 8, 128, 8));
  CRNN_TRY(make_tmap_nhwc_u8(&pl.qO_c32, pl.a3p, N, pl.H2, 4, 256, pl.mg3 ? 16 : 4));
  CRNN_TRY(make_tmap_nhwc_u8(&pl.qO_m42, pl.a4b, N, pl.H2, 2, 512, pl.mg4 ? 32 : 8));
  return CRNN_OK;
}

int fp8_conv2(crnn_model* m, convsw::Params p, bool lines, int sms, cudaStream_t st) {
  State* s = reinterpret_cast<State*>(m->fp8);
  const Plan& pl = m->plan;
  p.oscale = s->scales + 0;
  return launch_conv2_swap_lines<true>(lines, pl.tA_c2s, m->tB_c2, pl.qO_c2s, p, sms, st);
}

// layer 0 conv3_1 (EPI_RELU -> e4m3 a3), 1 conv3_2 (EPI_RELU_POOL12 -> e4m3 a3p), 2 / 3 conv4_1 / conv4_2 (EPI_STATS -> bf16 pre-BN;
// `moving`: with the moving statistics folded into colscale_m and p.bias, EPI_RELU -> e4m3 a4a / EPI_RELU_POOL12 -> e4m3 a4b);
// `p` is the bf16 path's conv_params (output, bias, stats, line widths), re-cut into 128-channel K-blocks here
int fp8_conv_gemm(crnn_model* m, int layer, gemm::Params p, bool lines, int sms, cudaStream_t st, bool moving) {
  State* s = reinterpret_cast<State*>(m->fp8);
  const Plan& pl = m->plan;
  p.cin_blocks = fp8::kL[layer].Cin / 128;
  p.num_k_blocks = 9 * p.cin_blocks;
  p.colscale = s->colscale + layer * 512;
  p.oscale = s->scales + layer + 1;
  const CUtensorMap* tA[4] = {&pl.q_c31, &pl.q_c32, &pl.q_c41, &pl.q_c42};
  const CUtensorMap* tO[4] = {&pl.q_c32, &pl.qO_c32, &pl.tO_c41, &pl.tO_c42};
  const CUtensorMap& a = *tA[layer];
  const CUtensorMap& b = s->tB[layer];
  using namespace gemm;
  if (moving) {
    p.colscale = s->colscale_m + (layer - 2) * 512;
    if (layer == 2) return launch_gemm_lines<256, A_CONV3, EPI_RELU, 4, 2>(lines, a, b, p, sms, st, &pl.q_c42);
    return launch_gemm_lines<256, A_CONV3, EPI_RELU_POOL12, 4, 2>(lines, a, b, p, sms, st, &pl.qO_m42);
  }
  switch (layer) {
    case 0: return launch_gemm_lines<256, A_CONV3, EPI_RELU, 4, 2>(lines, a, b, p, sms, st, tO[0]);
    case 1: return launch_gemm_lines<256, A_CONV3, EPI_RELU_POOL12, 4, 2>(lines, a, b, p, sms, st, tO[1]);
    default: return launch_gemm_lines<256, A_CONV3, EPI_STATS, 4, 2>(lines, a, b, p, sms, st, tO[layer]);
  }
}

// BatchNorm + ReLU of conv4_1 (layer 0: -> e4m3 a4a) or + pool3 of conv4_2 (layer 1: -> e4m3 a4b); bn = [4][512] or, lines, [N][4][512]
int fp8_bn_apply(crnn_model* m, int layer, const float* bn, bool lines, cudaStream_t st) {
  State* s = reinterpret_cast<State*>(m->fp8);
  const Plan& pl = m->plan;
  const int Wo = layer ? 2 : 4;
  const size_t nvec = (size_t)pl.N * pl.H2 * Wo * 512 / 8;
  const unsigned grid = (unsigned)((nvec + 255) / 256);
  const uint4* in = reinterpret_cast<const uint4*>(layer ? pl.a4b_pre : pl.a4a_pre);
  uint2* out = reinterpret_cast<uint2*>(layer ? pl.a4b : pl.a4a);
  const float* os = s->scales + 3 + layer;
  using fp8::bn_apply_e4m3_kernel;
  const auto kern = layer ? (lines ? bn_apply_e4m3_kernel<true, true> : bn_apply_e4m3_kernel<true, false>)
                          : (lines ? bn_apply_e4m3_kernel<false, true> : bn_apply_e4m3_kernel<false, false>);
  kern<<<grid, 256, 0, st>>>(in, out, bn, lines ? pl.line_w : nullptr, os, nvec, pl.H2, Wo, 512);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}

// conv5 (2x2 VALID) over the e4m3 [N*H2, 2 x 512] rows: 8 K-blocks per row shift, bf16 output as on the bf16 path
int fp8_conv5(crnn_model* m, gemm::Params p, int sms, cudaStream_t st) {
  State* s = reinterpret_cast<State*>(m->fp8);
  p.kb_per_shift = 8;
  p.num_k_blocks = 16;
  p.colscale = s->colscale + 4 * 512;
  return launch_gemm<256, gemm::A_PLAIN, gemm::EPI_BIAS_BF16, 4, 2>(m->plan.q_c5, s->tB[4], p, sms, st, &m->plan.tA_x);
}

// after the bf16 front end of a calibration batch: amax of a2, a3, a3p, a4a, a4b -> power-of-two scales
int fp8_finish_calibration(crnn_model* m, cudaStream_t st) {
  State* s = reinterpret_cast<State*>(m->fp8);
  const Plan& pl = m->plan;
  const size_t pos = (size_t)pl.N * pl.H2;
  const struct { const __nv_bfloat16* p; size_t n; } t[fp8::kLayers] = {
      {pl.a2, pos * 8 * 128}, {pl.a3, pos * 8 * 256}, {pl.a3p, pos * 4 * 256}, {pl.a4a, pos * 4 * 512}, {pl.a4b, pos * 2 * 512}};
  CUDA_TRY(cudaMemsetAsync(s->amax, 0, fp8::kLayers * sizeof(unsigned), st));
  for (int l = 0; l < fp8::kLayers; ++l) {
    const size_t nvec = t[l].n / 8;
    size_t grid = (nvec + 255) / 256;
    if (grid > (size_t)m->num_sms * 8) grid = (size_t)m->num_sms * 8;
    fp8::amax_bf16_kernel<<<(unsigned)grid, 256, 0, st>>>(reinterpret_cast<const uint4*>(t[l].p), nvec, s->amax + l);
    CUDA_TRY(cudaGetLastError());
  }
  fp8::scale_finalize_kernel<<<1, 32, 0, st>>>(s->amax, s->scales);
  CUDA_TRY(cudaGetLastError());
  s->calibrated = true;
  s->colscale_dirty = true;
  return CRNN_OK;
}

int fp8_get_scales(crnn_model* m, float* host) {
  State* s = reinterpret_cast<State*>(m->fp8);
  if (!s || !s->calibrated) return crnn_fail(CRNN_INVALID_VALUE, "get_fp8_scales: the fp8 model is not calibrated (crnn_model_calibrate_fp8 or crnn_model_set_fp8_scales)");
  CUDA_TRY(cudaDeviceSynchronize());
  CUDA_TRY(cudaMemcpy(host, s->scales, fp8::kLayers * sizeof(float), cudaMemcpyDeviceToHost));
  return CRNN_OK;
}

int fp8_set_scales(crnn_model* m, const float* host) {
  for (int l = 0; l < fp8::kLayers; ++l) {
    int e = 0;
    const float v = host[l];
    if (!(v > 0.f) || !std::isfinite(v) || std::frexp(v, &e) != 0.5f || e - 1 < -126)
      return crnn_fail(CRNN_INVALID_VALUE, "set_fp8_scales: scale %d = %g is not a power of two in [2^-126, 2^127]", l, (double)v);
  }
  State* s = reinterpret_cast<State*>(m->fp8);
  CUDA_TRY(cudaDeviceSynchronize());     // a calibration still queued on some stream must not overwrite these afterwards
  CUDA_TRY(cudaMemcpy(s->scales, host, fp8::kLayers * sizeof(float), cudaMemcpyHostToDevice));
  // a copy from pageable memory may return before its DMA lands, and the next forward may run on a non-blocking stream
  CUDA_TRY(cudaDeviceSynchronize());
  s->calibrated = true;
  s->colscale_dirty = true;
  return CRNN_OK;
}

// crnn_debug_tap of an fp8 activation: index 0..4 = a2, a3, a3p, a4a, a4b
int fp8_dequant_tap(crnn_model* m, int idx, const void* src, float* dst, size_t n, cudaStream_t st) {
  State* s = reinterpret_cast<State*>(m->fp8);
  fp8::dequant_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(reinterpret_cast<const uint8_t*>(src), s->scales + idx, dst, n);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}

// crnn_debug_tap_raw names of the fp8 state: "fp8_scales" f32 [5], "fp8_colscale" f32 [5][512], "fp8_colscale_moving" f32 [2][512],
// "fp8_wscale" f32 [5][512],
// "fp8_w_<layer>" u8 [Cout][K].  Returns 1 when `name` is one of them (the copy is issued or has failed with a status in *status).
int fp8_debug_tap_raw(crnn_model* m, const std::string& name, void* dst, size_t dst_bytes, cudaStream_t st, int* status) {
  State* s = reinterpret_cast<State*>(m->fp8);
  const void* src = nullptr;
  size_t bytes = 0;
  if (name == "fp8_scales") { bytes = fp8::kLayers * sizeof(float); src = s ? s->scales : nullptr; }
  else if (name == "fp8_colscale") { bytes = fp8::kLayers * 512 * sizeof(float); src = s ? s->colscale : nullptr; }
  else if (name == "fp8_colscale_moving") { bytes = 2 * 512 * sizeof(float); src = s ? s->colscale_m : nullptr; }
  else if (name == "fp8_wscale") { bytes = fp8::kLayers * 512 * sizeof(float); src = s ? s->wscale : nullptr; }
  else {
    for (int l = 0; l < fp8::kLayers; ++l)
      if (name == std::string("fp8_w_") + fp8::kL[l].name) { bytes = (size_t)fp8::kL[l].K * fp8::kL[l].Cout; src = s ? s->Wq[l] : nullptr; }
    if (bytes == 0) return 0;
  }
  if (src == nullptr) *status = crnn_fail(CRNN_INVALID_VALUE, "debug_tap_raw: %s: no fp8 forward or calibration ran yet", name.c_str());
  else if (dst_bytes < bytes) *status = crnn_fail(CRNN_INVALID_VALUE, "debug_tap_raw: dst too small (%zu < %zu bytes)", dst_bytes, bytes);
  else if (cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st) != cudaSuccess) *status = crnn_fail(CRNN_CUDA_ERROR, "debug_tap_raw: copy failed");
  else *status = CRNN_OK;
  return 1;
}
