// f32-class forward paths (crnn_config.compute_dtype = 2 and 3) -- BASELINE configs[1]: "fp32 CRNN fwd + CTC loss, batch 256, 32x160".
//
// The reference computes everything in fp32 (lib/networks/LSTM_train.py:10, network.py:166,174).  The tensor cores have no
// fp32 operand kind; the two ways to an fp32-class contraction are tf32 operands (10-bit mantissa: 8x finer than
// bf16, still 2^13 coarser than fp32) and the split-operand scheme used here ("3xbf16"), which keeps ~16 mantissa bits per
// operand and the f32 accumulator of the bf16 wgmma:
//
//      a = ah + al,  w = wh + wl   (ah = bf16(a), al = bf16(a - ah), same for w)
//      a*w ~= ah*wh + al*wh + ah*wl                      (the dropped al*wl term is 2^-18 relative)
//
// Every activation tensor is therefore stored as bf16 NHWC with 2C channels [hi(C) | lo(C)], every weight matrix as a K-major
// B operand with a tripled K = [wh | wh | wl], and the SAME wgmma/TMA implicit-GEMM kernels of gemm.cuh run over the virtual
// K = [hi | lo | hi] (the producer folds the third group back onto the hi half: gemm::Params::cin_phys / kb_phys).  The
// accumulators leave the GEMM as raw f32 (EPI_CONV_F32 / EPI_F32); bias, batch-stat BN (f64 sums), ReLU, the max-pools and
// the hi/lo split are done by the small HBM-bound kernels below in f32; conv1 (K = 9) runs as f32 FMAs; the LSTM cell uses
// expf/tanhf and an f32 input projection.  Measured against the fp64 oracle: tests/test_gpu_x3.py.
//
// compute_dtype = 3 runs the same orchestration with tf32 operands instead (template parameter TF of the kernels below,
// gemm::gemm_kernel<..., KIND = 1>): activations stay f32 NHWC with C channels (the same bytes as the [hi | lo] bf16 rows), weights
// are f32 K-major [Cout][K], both rounded to nearest tf32 where they are produced (the tensor core would truncate), 32 elements per
// 128 B K-block, one pass over K at half the bf16 rate.  Operand precision 2^-11 instead of 2^-17: the middle point between
// the bf16 throughput path and the split path, and the operand kind SURVEY 7.2(6) names for this configuration.
//
// This is the parity configuration (3x the MMA work, unfused elementwise passes, one GEMM + one cell launch per time step);
// the throughput configuration is the bf16 path of model.cu.  Forward + CTC only: no backward in this mode.
#include <cstring>
#include <string>

#include "gemm_launch.h"
#include "kernels.cuh"
#include "model_internal.h"

namespace x3 {

__device__ __forceinline__ void split2(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

__device__ __forceinline__ uint2 pack4(const __nv_bfloat16* h) {
  uint2 r;
  r.x = (uint32_t)__bfloat16_as_ushort(h[0]) | ((uint32_t)__bfloat16_as_ushort(h[1]) << 16);
  r.y = (uint32_t)__bfloat16_as_ushort(h[2]) | ((uint32_t)__bfloat16_as_ushort(h[3]) << 16);
  return r;
}

// ---- weights: dst[co][g*3*inner + part*inner + k] = part < 2 ? hi(src[(g*inner + k)*ld + co]) : lo(...)
__global__ void __launch_bounds__(256) split_weight_kernel(const float* __restrict__ src, int K, int Cout, int ld, int inner,
                                                           __nv_bfloat16* __restrict__ dst) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)K * Cout) return;
  const int r = (int)(i / Cout), co = (int)(i - (size_t)r * Cout);
  const int g = r / inner, k = r - g * inner;
  __nv_bfloat16 hi, lo;
  split2(__ldg(src + (size_t)r * ld + co), hi, lo);
  __nv_bfloat16* d = dst + (size_t)co * 3 * K + (size_t)g * 3 * inner + k;
  d[0] = hi; d[inner] = hi; d[2 * inner] = lo;
}

// ---- tf32 weights: dst[co][r] = tf32(src[r*ld + co])  (K-major B operand, natural K order)
__global__ void __launch_bounds__(256) tf32_weight_kernel(const float* __restrict__ src, int K, int Cout, int ld, float* __restrict__ dst) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)K * Cout) return;
  const int r = (int)(i / Cout), co = (int)(i - (size_t)r * Cout);
  dst[(size_t)co * K + r] = ptx::round_tf32(__ldg(src + (size_t)r * ld + co));
}

// Store 4 consecutive channels of one activation position: split mode writes the hi quad at `o` and the lo quad `lo_off`
// elements later (bf16); tf32 mode writes one float4 of tf32-rounded values.
template <bool TF>
__device__ __forceinline__ void store_quad(void* base, size_t off, size_t lo_off, const float (&v)[4]) {
  if constexpr (TF) {
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + off) =
        make_float4(ptx::round_tf32(v[0]), ptx::round_tf32(v[1]), ptx::round_tf32(v[2]), ptx::round_tf32(v[3]));
  } else {
    __nv_bfloat16 hi[4], lo[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) split2(v[j], hi[j], lo[j]);
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(base) + off;
    *reinterpret_cast<uint2*>(o) = pack4(hi);
    *reinterpret_cast<uint2*>(o + lo_off) = pack4(lo);
  }
}

// ---- conv1 (3x3 SAME, 1 -> 64) + bias + ReLU + pool1 (2x2/2), f32 FMAs, hi/lo output [N, W/2, 16, 128]
//      (lib/networks/LSTM_train.py:24-25).  One thread per (pooled position, 4 channels).  TIn: float (the f32 data tensor) or
//      uint8_t (pixel bytes, widened at the load to the same f32 values: common.cuh)
template <bool TF, typename TIn = float>
__global__ void __launch_bounds__(256) conv1_kernel(const TIn* __restrict__ data, const float* __restrict__ wgt,
                                                    const float* __restrict__ bias, void* __restrict__ out, int N, int W) {
  const int H1 = W >> 1;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)N * H1 * 16 * 16;
  if (i >= total) return;
  const int c4 = (int)(i & 15);
  const size_t pos = i >> 4;
  const int wo = (int)(pos & 15);
  const int ho = (int)((pos >> 4) % H1);
  const int n = (int)((pos >> 4) / H1);
  float patch[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int gr = 2 * ho - 1 + a, gc = 2 * wo - 1 + b;
      patch[a][b] = (gr >= 0 && gr < W && gc >= 0 && gc < 32) ? pixel_f32(__ldg(data + ((size_t)n * W + gr) * 32 + gc)) : 0.f;
    }
  float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
#pragma unroll
  for (int dy = 0; dy < 2; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const float4 w4 = __ldg(reinterpret_cast<const float4*>(wgt + (r * 3 + s) * 64 + c4 * 4));
          const float x = patch[dy + r][dx + s];
          acc[0] = fmaf(x, w4.x, acc[0]); acc[1] = fmaf(x, w4.y, acc[1]); acc[2] = fmaf(x, w4.z, acc[2]); acc[3] = fmaf(x, w4.w, acc[3]);
        }
#pragma unroll
      for (int j = 0; j < 4; ++j) best[j] = fmaxf(best[j], acc[j]);
    }
  const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + c4 * 4));
  const float v[4] = {fmaxf(best[0] + b4.x, 0.f), fmaxf(best[1] + b4.y, 0.f), fmaxf(best[2] + b4.z, 0.f), fmaxf(best[3] + b4.w, 0.f)};
  store_quad<TF>(out, pos * (TF ? 64 : 128) + c4 * 4, 64, v);
}

// ---- f32 NHWC [Nimg, H, Wd, C] -> (+bias) -> (BN scale/shift) -> (ReLU) -> (max-pool) -> hi/lo bf16
// POOL: 0 none, 1 = 2x2/2 over (H, Wd), 2 = 1x2 over Wd (network.py:343-350: ksize [1,k_h,k_w,1] on [N, width, height, C]).
// Output layout: groups of G consecutive output positions share one row [hi(G*C) | lo(G*C)]  (G = 1: NHWC with 2C channels;
// G = 2: the [N*H2, (2 x 512) | (2 x 512)] rows conv5's row-shift GEMM reads).  One thread per (output position, 4 channels).
template <int POOL, bool TF>
__global__ void __launch_bounds__(256) act_split_kernel(const float* __restrict__ in, void* __restrict__ out,
                                                        const float* __restrict__ bias, const float* __restrict__ scale,
                                                        const float* __restrict__ shift, int relu, int Nimg, int H, int Wd, int C,
                                                        int G) {
  const int Ho = (POOL == 1) ? (H >> 1) : H, Wo = (POOL != 0) ? (Wd >> 1) : Wd;
  const int c4n = C >> 2;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)Nimg * Ho * Wo * c4n;
  if (i >= total) return;
  const int c = (int)(i % c4n) * 4;
  const size_t pos = i / c4n;
  const int wo = (int)(pos % Wo);
  const int ho = (int)((pos / Wo) % Ho);
  const int n = (int)(pos / ((size_t)Wo * Ho));
  const float4 b4 = bias ? __ldg(reinterpret_cast<const float4*>(bias + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
  const float4 s4 = scale ? __ldg(reinterpret_cast<const float4*>(scale + c)) : make_float4(1.f, 1.f, 1.f, 1.f);
  const float4 h4 = shift ? __ldg(reinterpret_cast<const float4*>(shift + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
  float v[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
  const int ny = (POOL == 1) ? 2 : 1, nx = (POOL != 0) ? 2 : 1;
  for (int dy = 0; dy < ny; ++dy)
    for (int dx = 0; dx < nx; ++dx) {
      const int hh = (POOL == 1) ? 2 * ho + dy : ho, ww = (POOL != 0) ? 2 * wo + dx : wo;
      const float4 x = __ldg(reinterpret_cast<const float4*>(in + (((size_t)n * H + hh) * Wd + ww) * C + c));
      float y[4] = {fmaf(x.x + b4.x, s4.x, h4.x), fmaf(x.y + b4.y, s4.y, h4.y), fmaf(x.z + b4.z, s4.z, h4.z), fmaf(x.w + b4.w, s4.w, h4.w)};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (relu) y[j] = fmaxf(y[j], 0.f);
        v[j] = fmaxf(v[j], y[j]);
      }
    }
  if constexpr (TF) store_quad<true>(out, pos * (size_t)C + c, 0, v);        // plain NHWC: G consecutive positions are already one row
  else store_quad<false>(out, (pos / G) * (size_t)(2 * G * C) + (pos % G) * (size_t)C + c, (size_t)G * C, v);
}

// ---- per-channel sum / sum of squares of (x + bias) over P positions, f64 (batch-stat BN, network.py:177-178)
__global__ void __launch_bounds__(256) bn_stats_kernel(const float* __restrict__ in, const float* __restrict__ bias, size_t P, int C,
                                                       double* __restrict__ stats) {
  const int c4n = C >> 2;                                   // C = 512 -> 128 channel quads, 2 positions per 256-thread pass
  const int cq = threadIdx.x % c4n, sub = threadIdx.x / c4n, per = blockDim.x / c4n;
  const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + cq * 4));
  double s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
  for (size_t p = (size_t)blockIdx.x * per + sub; p < P; p += (size_t)gridDim.x * per) {
    const float4 x = __ldg(reinterpret_cast<const float4*>(in + p * C + cq * 4));
    const double a = (double)(x.x + b4.x), b = (double)(x.y + b4.y), c = (double)(x.z + b4.z), d = (double)(x.w + b4.w);
    s[0] += a; s[1] += b; s[2] += c; s[3] += d;
    q[0] += a * a; q[1] += b * b; q[2] += c * c; q[3] += d * d;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    atomicAdd(stats + cq * 4 + j, s[j]);
    atomicAdd(stats + C + cq * 4 + j, q[j]);
  }
}

// ---- LSTM cell for one time step, both directions (network.py:98-109; TF LSTMCell: gates i,j,f,o, forget_bias 1.0, state
// carried and output zero past sequence_length, backward direction = reverse_sequence by length).  One thread per (dir, n, unit).
//   z     [2*Npad, 2048] f32   h_{t-1} W_h for both weight sets (row block d uses columns d*1024 ..)
//   xproj [N*H, 2048]    f32   x_t W_x (no bias), natural gate order per direction
//   hS    [2*Npad, 512]  bf16  hi | lo of h (A operand of the next step)
//   lo    [N*H, 1024]    bf16  lstm_out, hi(fw 256, bw 256) | lo(..) (A operand of the 512 -> 64 projection)
// tf32 mode: hS [2*Npad, 256] f32 and lo [N*H, 512] f32, tf32-rounded.
template <bool TF>
__global__ void __launch_bounds__(256) lstm_cell_kernel(const float* __restrict__ z, const float* __restrict__ xproj,
                                                        const float* __restrict__ b_fw, const float* __restrict__ b_bw,
                                                        float* __restrict__ cst, void* __restrict__ hS_, void* __restrict__ lo_,
                                                        const int* __restrict__ seq_len, int step, int Nimg, int Npad, int H, int T) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)2 * Nimg * 256) return;
  const int u = (int)(i & 255);
  const int n = (int)((i >> 8) % Nimg);
  const int dir = (int)((i >> 8) / Nimg);
  const int len = min(max(__ldg(seq_len + n), 0), T);
  if (step >= len) return;
  const int t = dir ? (len - 1 - step) : step;
  const size_t row = (size_t)dir * Npad + n;
  const float* zr = z + row * 2048 + dir * 1024 + u;
  const float* xr = xproj + ((size_t)n * H + t) * 2048 + dir * 1024 + u;
  const float* br = (dir ? b_bw : b_fw) + u;
  const float zi = zr[0] + __ldg(xr) + __ldg(br);
  const float zj = zr[256] + __ldg(xr + 256) + __ldg(br + 256);
  const float zf = zr[512] + __ldg(xr + 512) + __ldg(br + 512) + 1.0f;
  const float zo = zr[768] + __ldg(xr + 768) + __ldg(br + 768);
  const float si = 1.f / (1.f + expf(-zi)), sf = 1.f / (1.f + expf(-zf)), so = 1.f / (1.f + expf(-zo));
  float* cp = cst + row * 256 + u;
  const float c = sf * (*cp) + si * tanhf(zj);
  *cp = c;
  const float h = so * tanhf(c);
  if constexpr (TF) {
    const float hr = ptx::round_tf32(h);
    reinterpret_cast<float*>(hS_)[row * 256 + u] = hr;
    reinterpret_cast<float*>(lo_)[((size_t)n * H + t) * 512 + dir * 256 + u] = hr;
  } else {
    __nv_bfloat16* hS = reinterpret_cast<__nv_bfloat16*>(hS_);
    __nv_bfloat16 hh, hl;
    split2(h, hh, hl);
    hS[row * 512 + u] = hh;
    hS[row * 512 + 256 + u] = hl;
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(lo_) + ((size_t)n * H + t) * 1024 + dir * 256 + u;
    o[0] = hh;
    o[512] = hl;
  }
}

// ---- parity taps: hi/lo rows -> f32 (same G convention as act_split_kernel)
__global__ void split_to_f32_kernel(const __nv_bfloat16* __restrict__ in, float* __restrict__ out, size_t npos, int C, int G) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npos * C) return;
  const size_t pos = i / C;
  const int c = (int)(i - pos * C);
  const __nv_bfloat16* p = in + (pos / G) * (size_t)(2 * G * C) + (pos % G) * (size_t)C + c;
  out[i] = __bfloat162float(p[0]) + __bfloat162float(p[(size_t)G * C]);
}

struct Plan {
  int N = 0, W = 0, H1 = 0, H2 = 0, T = 0, Npad = 0;
  void* ws = nullptr;
  float *scratch, *xproj, *z, *cst;
  // activations: bf16 [hi | lo] rows (split mode) or f32 rows (tf32 mode) -- the same number of bytes either way
  uint8_t *s1, *s2, *s3, *s3p, *s4a, *s4b, *s5, *slo, *hS;
  double* stats;
  float* bn;
  int mg2, mg3, mg4;
  CUtensorMap tA_c2, tA_c31, tA_c32, tA_c41, tA_c42, tA_c5, tA_x, tA_l, tA_h;
};

struct State {
  bool tf32 = false;         // compute_dtype 3: tf32 operands
  void* wblock = nullptr;
  uint8_t *Bc2, *Bc31, *Bc32, *Bc41, *Bc42, *Bc5, *Bx, *Bh, *Bl;
  CUtensorMap tB_c2, tB_c31, tB_c32, tB_c41, tB_c42, tB_c5, tB_x, tB_h, tB_l;
  bool dirty = true;
  bool maps_ready = false;
  Plan plan;
};

static size_t layout(Plan& pl, int N, int W, uint8_t* base) {
  pl.N = N; pl.W = W; pl.H1 = W / 2; pl.H2 = W / 4; pl.T = W / 4 - 1;
  pl.Npad = (N + 127) / 128 * 128;
  size_t off = 0;
  auto take = [&](size_t bytes) { uint8_t* p = base ? base + off : nullptr; off += align_up(bytes); return p; };
  const size_t n = N, h1 = pl.H1, h2 = pl.H2;
  pl.scratch = (float*)take(n * h1 * 16 * 128 * 4);                 // largest raw f32 GEMM output (conv2)
  pl.s1 = take(n * h1 * 16 * 128 * 2);
  pl.s2 = take(n * h2 * 8 * 256 * 2);
  pl.s3 = take(n * h2 * 8 * 512 * 2);
  pl.s3p = take(n * h2 * 4 * 512 * 2);
  pl.s4a = take(n * h2 * 4 * 1024 * 2);
  pl.s4b = take(n * h2 * 2048 * 2);
  pl.s5 = take(n * h2 * 1024 * 2);
  pl.xproj = (float*)take(n * h2 * 2048 * 4);
  pl.slo = take(n * h2 * 1024 * 2);
  pl.z = (float*)take((size_t)2 * pl.Npad * 2048 * 4);
  pl.hS = take((size_t)2 * pl.Npad * 512 * 2);
  pl.cst = (float*)take((size_t)2 * pl.Npad * 256 * 4);
  pl.stats = (double*)take(2 * 2 * 512 * 8);
  pl.bn = (float*)take(2 * 4 * 512 * 4);
  return off;
}

static int build_plan(State* s, int N, int W, void* ws) {
  x3::Plan& pl = s->plan;
  layout(pl, N, W, reinterpret_cast<uint8_t*>(ws));
  pl.ws = ws;
  pl.mg2 = (pl.H1 % 8) == 0; pl.mg3 = (pl.H2 % 16) == 0; pl.mg4 = (pl.H2 % 32) == 0;
  if (s->tf32) {
    CRNN_TRY(make_tmap_nhwc_f32(&pl.tA_c2, pl.s1, N, pl.H1, 16, 64, pl.mg2 ? 8 : 2));
    CRNN_TRY(make_tmap_nhwc_f32(&pl.tA_c31, pl.s2, N, pl.H2, 8, 128, pl.mg3 ? 16 : 4));
    CRNN_TRY(make_tmap_nhwc_f32(&pl.tA_c32, pl.s3, N, pl.H2, 8, 256, pl.mg3 ? 16 : 4));
    CRNN_TRY(make_tmap_nhwc_f32(&pl.tA_c41, pl.s3p, N, pl.H2, 4, 256, pl.mg4 ? 32 : 8));
    CRNN_TRY(make_tmap_nhwc_f32(&pl.tA_c42, pl.s4a, N, pl.H2, 4, 512, pl.mg4 ? 32 : 8));
    const uint64_t Rt = (uint64_t)N * pl.H2;
    CRNN_TRY(make_tmap_2d_f32(&pl.tA_c5, pl.s4b, Rt, 1024, 1024, 128));
    CRNN_TRY(make_tmap_2d_f32(&pl.tA_x, pl.s5, Rt, 512, 512, 128));
    CRNN_TRY(make_tmap_2d_f32(&pl.tA_l, pl.slo, Rt, 512, 512, 128));
    CRNN_TRY(make_tmap_2d_f32(&pl.tA_h, pl.hS, (uint64_t)2 * pl.Npad, 256, 256, 128));
    return CRNN_OK;
  }
  CRNN_TRY(make_tmap_nhwc(&pl.tA_c2, pl.s1, N, pl.H1, 16, 128, pl.mg2 ? 8 : 2));
  CRNN_TRY(make_tmap_nhwc(&pl.tA_c31, pl.s2, N, pl.H2, 8, 256, pl.mg3 ? 16 : 4));
  CRNN_TRY(make_tmap_nhwc(&pl.tA_c32, pl.s3, N, pl.H2, 8, 512, pl.mg3 ? 16 : 4));
  CRNN_TRY(make_tmap_nhwc(&pl.tA_c41, pl.s3p, N, pl.H2, 4, 512, pl.mg4 ? 32 : 8));
  CRNN_TRY(make_tmap_nhwc(&pl.tA_c42, pl.s4a, N, pl.H2, 4, 1024, pl.mg4 ? 32 : 8));
  const uint64_t R = (uint64_t)N * pl.H2;
  CRNN_TRY(make_tmap_2d(&pl.tA_c5, pl.s4b, R, 2048, 2048, 128));
  CRNN_TRY(make_tmap_2d(&pl.tA_x, pl.s5, R, 1024, 1024, 128));
  CRNN_TRY(make_tmap_2d(&pl.tA_l, pl.slo, R, 1024, 1024, 128));
  CRNN_TRY(make_tmap_2d(&pl.tA_h, pl.hS, (uint64_t)2 * pl.Npad, 512, 512, 128));
  return CRNN_OK;
}

static int prepare(crnn_model* m, State* s, cudaStream_t st) {
  const int kK[9] = {576, 1152, 2304, 2304, 4608, 2048, 512, 256, 512};            // contraction length per layer
  const int kCo[9] = {128, 256, 256, 512, 512, 512, 2048, 2048, 64};
  if (!s->wblock) {
    // bytes per weight element: 3 bf16 parts (split) or one f32 (tf32)
    const size_t eb = s->tf32 ? 4 : 6;
    size_t tot = 0;
    for (int i = 0; i < 9; ++i) tot += align_up((size_t)kK[i] * kCo[i] * eb);
    CUDA_TRY(cudaMalloc(&s->wblock, tot));
    uint8_t* p = reinterpret_cast<uint8_t*>(s->wblock);
    uint8_t** dst[9] = {&s->Bc2, &s->Bc31, &s->Bc32, &s->Bc41, &s->Bc42, &s->Bc5, &s->Bx, &s->Bh, &s->Bl};
    for (int i = 0; i < 9; ++i) { *dst[i] = p; p += align_up((size_t)kK[i] * kCo[i] * eb); }
  }
  if (s->tf32) {
    if (!s->maps_ready) {
      CUtensorMap* tm[9] = {&s->tB_c2, &s->tB_c31, &s->tB_c32, &s->tB_c41, &s->tB_c42, &s->tB_c5, &s->tB_x, &s->tB_h, &s->tB_l};
      uint8_t* base[9] = {s->Bc2, s->Bc31, s->Bc32, s->Bc41, s->Bc42, s->Bc5, s->Bx, s->Bh, s->Bl};
      const int box[9] = {128, 256, 256, 256, 256, 256, 256, 256, 64};
      for (int i = 0; i < 9; ++i) CRNN_TRY(make_tmap_2d_f32(tm[i], base[i], kCo[i], kK[i], kK[i], box[i]));
      s->maps_ready = true;
    }
    auto tw = [&](const float* src, int K, int Cout, int ld, uint8_t* dst) -> int {
      const size_t n = (size_t)K * Cout;
      tf32_weight_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, K, Cout, ld, reinterpret_cast<float*>(dst));
      CUDA_TRY(cudaGetLastError());
      return CRNN_OK;
    };
    CRNN_TRY(tw(m->P("conv2/weights"), 576, 128, 128, s->Bc2));
    CRNN_TRY(tw(m->P("conv3_1/weights"), 1152, 256, 256, s->Bc31));
    CRNN_TRY(tw(m->P("conv3_2/weights"), 2304, 256, 256, s->Bc32));
    CRNN_TRY(tw(m->P("conv4_1/weights"), 2304, 512, 512, s->Bc41));
    CRNN_TRY(tw(m->P("conv4_2/weights"), 4608, 512, 512, s->Bc42));
    CRNN_TRY(tw(m->P("conv5/weights"), 2048, 512, 512, s->Bc5));
    const char* dn[2] = {"logits/bidirectional_rnn/fw/lstm_cell/weights", "logits/bidirectional_rnn/bw/lstm_cell/weights"};
    for (int d = 0; d < 2; ++d) {
      const float* w = m->P(dn[d]);                                             // [768,1024], rows [x(512); h(256)]
      CRNN_TRY(tw(w, 512, 1024, 1024, s->Bx + (size_t)d * 1024 * 512 * 4));
      CRNN_TRY(tw(w + 512 * 1024, 256, 1024, 1024, s->Bh + (size_t)d * 1024 * 256 * 4));
    }
    CRNN_TRY(tw(m->P("logits/weights"), 512, 64, 64, s->Bl));
    s->dirty = false;
    return CRNN_OK;
  }
  if (!s->maps_ready) {
    s->maps_ready = true;
    CRNN_TRY(make_tmap_2d(&s->tB_c2, s->Bc2, 128, 1728, 1728, 128));
    CRNN_TRY(make_tmap_2d(&s->tB_c31, s->Bc31, 256, 3456, 3456, 256));
    CRNN_TRY(make_tmap_2d(&s->tB_c32, s->Bc32, 256, 6912, 6912, 256));
    CRNN_TRY(make_tmap_2d(&s->tB_c41, s->Bc41, 512, 6912, 6912, 256));
    CRNN_TRY(make_tmap_2d(&s->tB_c42, s->Bc42, 512, 13824, 13824, 256));
    CRNN_TRY(make_tmap_2d(&s->tB_c5, s->Bc5, 512, 6144, 6144, 256));
    CRNN_TRY(make_tmap_2d(&s->tB_x, s->Bx, 2048, 1536, 1536, 256));
    CRNN_TRY(make_tmap_2d(&s->tB_h, s->Bh, 2048, 768, 768, 256));
    CRNN_TRY(make_tmap_2d(&s->tB_l, s->Bl, 64, 1536, 1536, 64));
  }
  auto sw = [&](const float* src, int K, int Cout, int ld, int inner, uint8_t* dst) -> int {
    const size_t n = (size_t)K * Cout;
    split_weight_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, K, Cout, ld, inner, reinterpret_cast<__nv_bfloat16*>(dst));
    CUDA_TRY(cudaGetLastError());
    return CRNN_OK;
  };
  CRNN_TRY(sw(m->P("conv2/weights"), 576, 128, 128, 64, s->Bc2));
  CRNN_TRY(sw(m->P("conv3_1/weights"), 1152, 256, 256, 128, s->Bc31));
  CRNN_TRY(sw(m->P("conv3_2/weights"), 2304, 256, 256, 256, s->Bc32));
  CRNN_TRY(sw(m->P("conv4_1/weights"), 2304, 512, 512, 256, s->Bc41));
  CRNN_TRY(sw(m->P("conv4_2/weights"), 4608, 512, 512, 512, s->Bc42));
  CRNN_TRY(sw(m->P("conv5/weights"), 2048, 512, 512, 1024, s->Bc5));        // groups = kh (row shift), inner = (kw, ci)
  const char* dirs[2] = {"logits/bidirectional_rnn/fw/lstm_cell/weights", "logits/bidirectional_rnn/bw/lstm_cell/weights"};
  for (int d = 0; d < 2; ++d) {
    const float* w = m->P(dirs[d]);                                             // [768,1024], rows [x(512); h(256)]
    CRNN_TRY(sw(w, 512, 1024, 1024, 512, s->Bx + (size_t)d * 1024 * 1536 * 2));
    CRNN_TRY(sw(w + 512 * 1024, 256, 1024, 1024, 256, s->Bh + (size_t)d * 1024 * 768 * 2));
  }
  CRNN_TRY(sw(m->P("logits/weights"), 512, 64, 64, 512, s->Bl));
  s->dirty = false;
  return CRNN_OK;
}

template <int POOL>
static int act_split(bool tf, const float* in, void* out, const float* bias, const float* scale, const float* shift, int relu, int Nimg,
                     int H, int Wd, int C, int G, cudaStream_t st) {
  const int Ho = (POOL == 1) ? H / 2 : H, Wo = (POOL != 0) ? Wd / 2 : Wd;
  const size_t total = (size_t)Nimg * Ho * Wo * (C / 4);
  const unsigned grid = (unsigned)((total + 255) / 256);
  if (tf) act_split_kernel<POOL, true><<<grid, 256, 0, st>>>(in, out, bias, scale, shift, relu, Nimg, H, Wd, C, G);
  else act_split_kernel<POOL, false><<<grid, 256, 0, st>>>(in, out, bias, scale, shift, relu, Nimg, H, Wd, C, G);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}

}  // namespace x3

// ------------------------------------------------------------------------------------------------ entry points (model.cu)
size_t x3_workspace_size(int N, int W) {
  x3::Plan pl;
  return x3::layout(pl, N, W, nullptr);
}

void x3_destroy(crnn_model* m) {
  x3::State* s = reinterpret_cast<x3::State*>(m->x3);
  if (!s) return;
  if (s->wblock) cudaFree(s->wblock);
  delete s;
  m->x3 = nullptr;
}

void x3_params_changed(crnn_model* m) {
  if (m->x3) reinterpret_cast<x3::State*>(m->x3)->dirty = true;
}

int x3_forward(crnn_model* m, const void* data, bool u8, const int* time_step_len, int N, int W, float* logits_out, void* workspace,
               size_t workspace_bytes, cudaStream_t st) {
  using namespace x3;
  if (!m->x3) {
    State* ns = new State();
    ns->tf32 = (m->cfg.compute_dtype == 3);
    m->x3 = ns;
  }
  State* s = reinterpret_cast<State*>(m->x3);
  const bool tf = s->tf32;
  if (workspace_bytes < x3_workspace_size(N, W)) return crnn_fail(CRNN_WORKSPACE_TOO_SMALL, "forward(f32 path): workspace too small");
  if (s->dirty) CRNN_TRY(prepare(m, s, st));
  x3::Plan& pl = s->plan;
  if (pl.N != N || pl.W != W || pl.ws != workspace) CRNN_TRY(build_plan(s, N, W, workspace));
  const int H1 = pl.H1, H2 = pl.H2, T = pl.T, sms = m->num_sms;
  const int R = N * H2;
  // K-blocks (128 B of operand) per 64 real input channels: 3 virtual bf16 blocks [hi | lo | hi] or 2 tf32 blocks
  const int kmul = tf ? 2 : 3;

  // conv1 + pool1 (f32 FMAs) -> s1 [N,H1,16, 64|64] (split) or [N,H1,16,64] f32 (tf32)
  {
    const size_t total = (size_t)N * H1 * 16 * 16;
    const unsigned grid = (unsigned)((total + 255) / 256);
    const float* wc = m->P("conv1/weights");
    const float* bc = m->P("conv1/biases");
    const float* df = static_cast<const float*>(data);
    const uint8_t* du = static_cast<const uint8_t*>(data);
    if (tf && u8) conv1_kernel<true, uint8_t><<<grid, 256, 0, st>>>(du, wc, bc, pl.s1, N, W);
    else if (tf) conv1_kernel<true><<<grid, 256, 0, st>>>(df, wc, bc, pl.s1, N, W);
    else if (u8) conv1_kernel<false, uint8_t><<<grid, 256, 0, st>>>(du, wc, bc, pl.s1, N, W);
    else conv1_kernel<false><<<grid, 256, 0, st>>>(df, wc, bc, pl.s1, N, W);
    CUDA_TRY(cudaGetLastError());
  }
  auto conv = [&](const CUtensorMap& ta, const CUtensorMap& tb, int H, int Wd, int Cin, int Cout, int merged, bool n128) -> int {
    gemm::Params p = conv_params(N, H, Wd, kmul * Cin, Cout, n128 ? 128 : 256, nullptr, pl.scratch, merged);
    p.cin_phys = tf ? 0 : 2 * Cin / 64;
    if (tf) {
      if (n128) return launch_gemm<128, gemm::A_CONV3, gemm::EPI_CONV_F32, 6, 1>(ta, tb, p, sms, st);
      return launch_gemm<256, gemm::A_CONV3, gemm::EPI_CONV_F32, 4, 1>(ta, tb, p, sms, st);
    }
    if (n128) return launch_gemm<128, gemm::A_CONV3, gemm::EPI_CONV_F32, 6>(ta, tb, p, sms, st);
    return launch_gemm<256, gemm::A_CONV3, gemm::EPI_CONV_F32, 4>(ta, tb, p, sms, st);
  };
  // plain GEMM [rows, K] x [Nc, K]^T -> f32; kreal = real contraction length per row shift, shifts = 1 (2 for conv5: rows m, m+1)
  auto plain = [&](const CUtensorMap& ta, const CUtensorMap& tb, int rows, int kreal, int shifts, int Nc, float* out) -> int {
    gemm::Params p;
    memset(&p, 0, sizeof(p));
    p.M = rows; p.num_m_tiles = (rows + 127) / 128; p.num_n_tiles = Nc / 256;
    p.kb_per_shift = kmul * kreal / 64; p.num_k_blocks = shifts * p.kb_per_shift; p.kb_phys = tf ? 0 : 2 * kreal / 64;
    p.row_shift_mul = 1; p.Nc = Nc; p.out = out;
    if (tf) return launch_gemm<256, gemm::A_PLAIN, gemm::EPI_F32, 4, 1>(ta, tb, p, sms, st);
    return launch_gemm<256, gemm::A_PLAIN, gemm::EPI_F32, 4>(ta, tb, p, sms, st);
  };
  // conv2 + ReLU + pool2 (2x2)
  CRNN_TRY(conv(pl.tA_c2, s->tB_c2, H1, 16, 64, 128, pl.mg2, true));
  CRNN_TRY(act_split<1>(tf, pl.scratch, pl.s2, m->P("conv2/biases"), nullptr, nullptr, 1, N, H1, 16, 128, 1, st));
  // conv3_1 + ReLU
  CRNN_TRY(conv(pl.tA_c31, s->tB_c31, H2, 8, 128, 256, pl.mg3, false));
  CRNN_TRY(act_split<0>(tf, pl.scratch, pl.s3, m->P("conv3_1/biases"), nullptr, nullptr, 1, N, H2, 8, 256, 1, st));
  // conv3_2 + ReLU + pool (1x2)
  CRNN_TRY(conv(pl.tA_c32, s->tB_c32, H2, 8, 256, 256, pl.mg3, false));
  CRNN_TRY(act_split<2>(tf, pl.scratch, pl.s3p, m->P("conv3_2/biases"), nullptr, nullptr, 1, N, H2, 8, 256, 1, st));
  // conv4_1 + batch-stat BN + ReLU
  CUDA_TRY(cudaMemsetAsync(pl.stats, 0, 2 * 2 * 512 * sizeof(double), st));
  const size_t P4 = (size_t)N * H2 * 4;
  CRNN_TRY(conv(pl.tA_c41, s->tB_c41, H2, 4, 256, 512, pl.mg4, false));
  bn_stats_kernel<<<2 * sms, 256, 0, st>>>(pl.scratch, m->P("conv4_1/biases"), P4, 512, pl.stats);
  CUDA_TRY(cudaGetLastError());
  CRNN_TRY(dp_allreduce_bn_finalize(m, pl.stats, (double)P4 * m->dp_world, m->P("conv4_1/conv4_1/gamma"), m->P("conv4_1/conv4_1/beta"),
                                    m->cfg.bn_eps, pl.bn, st));
  CRNN_TRY(act_split<0>(tf, pl.scratch, pl.s4a, m->P("conv4_1/biases"), pl.bn, pl.bn + 512, 1, N, H2, 4, 512, 1, st));
  // conv4_2 + BN + ReLU + pool3 (1x2) -> rows of two positions for conv5 ([hi(w0,w1) | lo(w0,w1)] in split mode)
  CRNN_TRY(conv(pl.tA_c42, s->tB_c42, H2, 4, 512, 512, pl.mg4, false));
  bn_stats_kernel<<<2 * sms, 256, 0, st>>>(pl.scratch, m->P("conv4_2/biases"), P4, 512, pl.stats + 1024);
  CUDA_TRY(cudaGetLastError());
  CRNN_TRY(dp_allreduce_bn_finalize(m, pl.stats + 1024, (double)P4 * m->dp_world, m->P("conv4_2/conv4_2/gamma"), m->P("conv4_2/conv4_2/beta"),
                                    m->cfg.bn_eps, pl.bn + 2048, st));
  CRNN_TRY(act_split<2>(tf, pl.scratch, pl.s4b, m->P("conv4_2/biases"), pl.bn + 2048, pl.bn + 2560, 1, N, H2, 4, 512, 2, st));
  // conv5 (2x2 VALID, no activation): rows m (kh = 0) and m+1 (kh = 1) of the [N*H2, 2 x 512] view
  CRNN_TRY(plain(pl.tA_c5, s->tB_c5, R, 1024, 2, 512, pl.scratch));
  CRNN_TRY(act_split<0>(tf, pl.scratch, pl.s5, m->P("conv5/biases"), nullptr, nullptr, 0, 1, R, 1, 512, 1, st));
  // LSTM input projection, both directions, f32 (bias is added by the cell)
  CRNN_TRY(plain(pl.tA_x, s->tB_x, R, 512, 1, 2048, pl.xproj));
  // recurrence: per step one GEMM (h x W_h, both weight sets) + one cell launch
  CUDA_TRY(cudaMemsetAsync(pl.hS, 0, (size_t)2 * pl.Npad * 512 * 2, st));
  CUDA_TRY(cudaMemsetAsync(pl.cst, 0, (size_t)2 * pl.Npad * 256 * 4, st));
  CUDA_TRY(cudaMemsetAsync(pl.slo, 0, (size_t)R * 1024 * 2, st));
  const float* b_fw = m->P("logits/bidirectional_rnn/fw/lstm_cell/biases");
  const float* b_bw = m->P("logits/bidirectional_rnn/bw/lstm_cell/biases");
  for (int step = 0; step < T; ++step) {
    CRNN_TRY(plain(pl.tA_h, s->tB_h, 2 * pl.Npad, 256, 1, 2048, pl.z));
    const size_t total = (size_t)2 * N * 256;
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (tf) lstm_cell_kernel<true><<<grid, 256, 0, st>>>(pl.z, pl.xproj, b_fw, b_bw, pl.cst, pl.hS, pl.slo, time_step_len, step, N, pl.Npad, H2, T);
    else lstm_cell_kernel<false><<<grid, 256, 0, st>>>(pl.z, pl.xproj, b_fw, b_bw, pl.cst, pl.hS, pl.slo, time_step_len, step, N, pl.Npad, H2, T);
    CUDA_TRY(cudaGetLastError());
  }
  // 512 -> 64 projection, time-major [T, N, 64] (network.py:126-128)
  {
    gemm::Params p;
    memset(&p, 0, sizeof(p));
    p.M = R; p.num_m_tiles = (R + 127) / 128; p.num_n_tiles = 1; p.num_k_blocks = kmul * 8; p.kb_per_shift = kmul * 8; p.kb_phys = tf ? 0 : 16;
    p.Nc = 64; p.bias = m->P("logits/biases"); p.out = logits_out; p.H = H2; p.T = T; p.Nimg = N;
    if (tf) CRNN_TRY((launch_gemm<64, gemm::A_PLAIN, gemm::EPI_LOGITS, 8, 1>(pl.tA_l, s->tB_l, p, sms, st)));
    else CRNN_TRY((launch_gemm<64, gemm::A_PLAIN, gemm::EPI_LOGITS, 8>(pl.tA_l, s->tB_l, p, sms, st)));
  }
  return CRNN_OK;
}

namespace x3 {
// activation buffer of a tap name: npos positions of C channels, G positions per [hi | lo] row (split mode)
static bool act_buffer(const Plan& pl, const std::string& k, const uint8_t** src, size_t* npos, int* C, int* G) {
  const size_t n = pl.N, h1 = pl.H1, h2 = pl.H2;
  *G = 1;
  if (k == "conv1") { *src = pl.s1; *npos = n * h1 * 16; *C = 64; }
  else if (k == "conv2") { *src = pl.s2; *npos = n * h2 * 8; *C = 128; }
  else if (k == "conv3_1") { *src = pl.s3; *npos = n * h2 * 8; *C = 256; }
  else if (k == "conv3_2") { *src = pl.s3p; *npos = n * h2 * 4; *C = 256; }
  else if (k == "conv4_1") { *src = pl.s4a; *npos = n * h2 * 4; *C = 512; }
  else if (k == "conv4_2") { *src = pl.s4b; *npos = n * h2 * 2; *C = 512; *G = 2; }
  else if (k == "conv5") { *src = pl.s5; *npos = n * h2; *C = 512; }
  else if (k == "lstm_out") { *src = pl.slo; *npos = n * h2; *C = 512; }
  else return false;
  return true;
}

static State* tapped_state(crnn_model* m, void* workspace) {
  State* s = reinterpret_cast<State*>(m->x3);
  return (!s || s->plan.ws == nullptr || s->plan.ws != workspace) ? nullptr : s;
}
}  // namespace x3

int x3_debug_tap(crnn_model* m, const char* name, float* dst, size_t dst_elems, void* workspace, cudaStream_t st) {
  using namespace x3;
  State* s = tapped_state(m, workspace);
  if (!s) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap: no forward ran on this workspace");
  x3::Plan& pl = s->plan;
  const std::string k(name);
  if (k == "xproj") {                 // f32 already, both directions in natural [i|j|f|o] order, no bias, rows not reversed
    const size_t cnt = (size_t)pl.N * pl.H2 * 2048;
    if (dst_elems < cnt) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap: dst too small");
    CUDA_TRY(cudaMemcpyAsync(dst, pl.xproj, cnt * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return CRNN_OK;
  }
  const uint8_t* src = nullptr;
  size_t npos = 0;
  int C = 0, G = 1;
  if (!act_buffer(pl, k, &src, &npos, &C, &G))
    return crnn_fail(CRNN_INVALID_VALUE, "debug_tap: %s does not exist on the f32-class paths (compute_dtype 2, 3)", name);
  if (dst_elems < npos * C) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap: dst too small");
  if (s->tf32) {
    CUDA_TRY(cudaMemcpyAsync(dst, src, npos * C * sizeof(float), cudaMemcpyDeviceToDevice, st));   // plain f32 NHWC already
    return CRNN_OK;
  }
  split_to_f32_kernel<<<(unsigned)((npos * C + 255) / 256), 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(src), dst, npos, C, G);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}

// Byte-for-byte copies of the f32-class workspace: "bn", "stats", "cst" and the activation buffers as stored (split mode:
// bf16 [hi | lo] rows, G positions per row; tf32 mode: f32 rows).  The same bytes per position in both modes.
int x3_debug_tap_raw(crnn_model* m, const char* name, void* dst, size_t dst_bytes, void* workspace, cudaStream_t st) {
  using namespace x3;
  State* s = tapped_state(m, workspace);
  if (!s) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap_raw: no forward ran on this workspace");
  x3::Plan& pl = s->plan;
  const std::string k(name);
  const void* src = nullptr;
  size_t bytes = 0;
  const uint8_t* act = nullptr;
  size_t npos = 0;
  int C = 0, G = 1;
  if (k == "bn") { src = pl.bn; bytes = 2 * 4 * 512 * sizeof(float); }
  else if (k == "stats") { src = pl.stats; bytes = 2 * 2 * 512 * sizeof(double); }
  else if (k == "cst") { src = pl.cst; bytes = (size_t)2 * pl.Npad * 256 * sizeof(float); }
  else if (act_buffer(pl, k, &act, &npos, &C, &G)) { src = act; bytes = npos * C * 4; }     // 2 x bf16 or 1 x f32 per value
  else return crnn_fail(CRNN_INVALID_VALUE, "debug_tap_raw: %s does not exist on the f32-class paths (compute_dtype 2, 3)", name);
  if (dst_bytes < bytes) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap_raw: dst too small (%zu < %zu bytes)", dst_bytes, bytes);
  CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st));
  return CRNN_OK;
}
