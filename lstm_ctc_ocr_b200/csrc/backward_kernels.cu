// HBM-bound kernels of the backward pass and the optimizer (everything that is not a tensor-core contraction).
// Restates the non-GEMM pieces of tf.gradients + tf.clip_by_global_norm + AdamOptimizer (lib/lstm/train.py:73-83).
#include "backward_kernels.cuh"

namespace {

__device__ __forceinline__ void unpack8(const uint4 q, float* v) {
  v[0] = ptx::bf16_lo(q.x); v[1] = ptx::bf16_hi(q.x); v[2] = ptx::bf16_lo(q.y); v[3] = ptx::bf16_hi(q.y);
  v[4] = ptx::bf16_lo(q.z); v[5] = ptx::bf16_hi(q.z); v[6] = ptx::bf16_lo(q.w); v[7] = ptx::bf16_hi(q.w);
}
__device__ __forceinline__ uint4 pack8(const float* v) {
  return make_uint4(ptx::pack_bf16x2(v[0], v[1]), ptx::pack_bf16x2(v[2], v[3]), ptx::pack_bf16x2(v[4], v[5]),
                    ptx::pack_bf16x2(v[6], v[7]));
}

// ---- d logits [T,N,64] f32 (time-major, already scaled by 1/N) -> rows (n,t) bf16 [N*H, 64]; rows t >= T are zero.
// Also the logits bias gradient (column sums).
__global__ void __launch_bounds__(256) dlogits_rows_kernel(const float* __restrict__ dlogits, __nv_bfloat16* __restrict__ rows,
                                                           float* __restrict__ dbias, int T, int N, int H) {
  __shared__ float red[64];
  if (threadIdx.x < 64) red[threadIdx.x] = 0.f;
  __syncthreads();
  const int c8 = threadIdx.x & 7;                    // 8 columns per thread
  float part[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) part[i] = 0.f;
  const long long total = (long long)N * H;
  for (long long r = (long long)blockIdx.x * 32 + (threadIdx.x >> 3); r < total; r += (long long)gridDim.x * 32) {
    const int n = (int)(r / H), t = (int)(r - (long long)n * H);
    float v[8];
    if (t < T) {
      const float4* src = reinterpret_cast<const float4*>(dlogits + ((size_t)t * N + n) * 64 + c8 * 8);
      const float4 a = __ldg(src), b = __ldg(src + 1);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = 0.f;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) part[i] += v[i];
    *reinterpret_cast<uint4*>(rows + r * 64 + c8 * 8) = pack8(v);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) atomicAdd(&red[c8 * 8 + i], part[i]);
  __syncthreads();
  if (threadIdx.x < 64) atomicAdd(dbias + threadIdx.x, red[threadIdx.x]);
}

// ---- column sums of a bf16 matrix [R, C] into f32 out[map(c)] (+=). perm_upc > 0: LSTM gate permutation inverse
// (two directions of 1024 permuted columns each -> TF column order, out has 2 x 1024 entries `dir_stride` apart).
// `mask` != nullptr: only elements whose mask value is > 0 count (the ReLU mask of a POOLED activation: the bias gradient of
// a conv followed by ReLU + max-pool is the column sum of the pooled gradient where the pooled output is positive -- every
// pooled gradient value is routed to exactly one pre-pool position -- so the 4x (2x) larger un-pooled tensor need not be re-read).
// `Cmod` > 0: the matrix is a [R, C] VIEW of a narrower [.., Cmod] tensor (Cmod divides C): column c accumulates into out[c % Cmod].
__global__ void __launch_bounds__(256) colsum_bf16_kernel(const __nv_bfloat16* __restrict__ src, const __nv_bfloat16* __restrict__ mask,
                                                          long long R, int C, int Cmod, float* __restrict__ out, int perm_upc,
                                                          long long dir_stride) {
  // block handles 256 columns (8 per thread x 32 lanes) x a strided set of rows (8 warps)
  const int cb = blockIdx.y * 256 + (threadIdx.x & 31) * 8;
  const bool okc = cb < C;
  float part[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) part[i] = 0.f;
  const long long stride = (long long)gridDim.x * 8;
  for (long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); r < R; r += 4 * stride) {
    uint4 q[4], mk[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long rr = r + u * stride;
      q[u] = (okc && rr < R) ? __ldg(reinterpret_cast<const uint4*>(src + rr * C + cb)) : make_uint4(0u, 0u, 0u, 0u);
      if (mask != nullptr) mk[u] = (okc && rr < R) ? __ldg(reinterpret_cast<const uint4*>(mask + rr * C + cb)) : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      float v[8];
      unpack8(q[u], v);
      if (mask != nullptr) {
        float y[8];
        unpack8(mk[u], y);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = (y[i] > 0.f) ? v[i] : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) part[i] += v[i];
    }
  }
  // block reduction over the 8 warps (same columns, different rows), then ONE atomic per column per block:
  // same-address f32 atomics from thousands of warps serialise in L2 and used to dominate this kernel
  __shared__ float red[8][256];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < 8; ++i) red[w][l * 8 + i] = part[i];
  __syncthreads();
  const int cl = threadIdx.x;                       // one column per thread
  const int c = blockIdx.y * 256 + cl;
  if (c < C) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k][cl];
    float* dst;
    if (perm_upc) {
      const int dir = c >> 10, pc = c & 1023;
      const int g = (pc % (4 * perm_upc)) / perm_upc, u = (pc / (4 * perm_upc)) * perm_upc + pc % perm_upc;
      dst = out + dir * dir_stride + g * 256 + u;
    } else {
      dst = out + (Cmod > 0 ? c % Cmod : c);
    }
    atomicAdd(dst, t);
  }
}

// ---- BatchNorm (+ReLU, + optional 1x2 max-pool) backward, pass 1 (sums only -- the routed gradient dy is NOT written here;
// pass 2 re-derives it from the same two inputs, which saves one 268 MB write + one 268 MB read per BN layer):
//   dy = routed upstream gradient at the pre-BN resolution, masked by ReLU;  sums[c] += dy, sums[C + c] += dy * xhat
// POOL = true (conv4_2 / pool3): dout is [P, Wp/2.., C] pooled; x_pre is [P*2 positions..]; the max is re-derived from
// the saved pre-BN tensor (first position wins ties).  POOL = false: dout has the same shape as x_pre (not launched: conv4_1's
// sums ride in conv4_2's data-gradient epilogue, gemm.cuh EPI_CONV_STORE_BNRED).
template <bool POOL>
__global__ void __launch_bounds__(256) bn_bwd_reduce_kernel(const uint4* __restrict__ dout, const uint4* __restrict__ x_pre,
                                                            uint4* __restrict__ dy, const float* __restrict__ bn /*scale,shift,mean,invstd*/,
                                                            double* __restrict__ sums, size_t out_positions, int C) {
  const int vpc = C / 8;
  const int cv = threadIdx.x % vpc;           // requires 256 % vpc == 0 (C = 512 -> vpc = 64)
  const int c = cv * 8;
  const int rows_per_block = 256 / vpc;
  float sc[8], sh[8], mu[8], is[8], s1[8], s2[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sc[i] = bn[c + i]; sh[i] = bn[C + c + i]; mu[i] = bn[2 * C + c + i]; is[i] = bn[3 * C + c + i];
    s1[i] = 0.f; s2[i] = 0.f;
  }
  // software-pipelined: the next position's 16-byte loads are in flight while this one is reduced (with one batch of loads
  // per iteration the pass is latency-bound at this occupancy)
  const size_t pstep = (size_t)gridDim.x * rows_per_block;
  size_t pos = (size_t)blockIdx.x * rows_per_block + threadIdx.x / vpc;
  uint4 qg = make_uint4(0u, 0u, 0u, 0u), qx0 = qg, qx1 = qg;
  if (pos < out_positions) {
    qg = __ldg(dout + pos * vpc + cv);
    qx0 = __ldg(x_pre + (POOL ? 2 * pos : pos) * vpc + cv);
    if (POOL) qx1 = __ldg(x_pre + (2 * pos + 1) * vpc + cv);
  }
  for (; pos < out_positions; pos += pstep) {
    const uint4 cg_ = qg, cx0 = qx0, cx1 = qx1;
    const size_t nxt = pos + pstep;
    if (nxt < out_positions) {
      qg = __ldg(dout + nxt * vpc + cv);
      qx0 = __ldg(x_pre + (POOL ? 2 * nxt : nxt) * vpc + cv);
      if (POOL) qx1 = __ldg(x_pre + (2 * nxt + 1) * vpc + cv);
    }
    float g[8];
    unpack8(cg_, g);
    if (POOL) {
      float x0[8], x1[8], d0[8], d1[8];
      unpack8(cx0, x0);
      unpack8(cx1, x1);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        // forward: bf16(relu(bn(x))) per position, then max; compare the same bf16-rounded values
        const float y0 = __bfloat162float(__float2bfloat16_rn(fmaxf(fmaf(x0[i], sc[i], sh[i]), 0.f)));
        const float y1 = __bfloat162float(__float2bfloat16_rn(fmaxf(fmaf(x1[i], sc[i], sh[i]), 0.f)));
        const bool first = (y0 >= y1);
        const float gy = ((first ? y0 : y1) > 0.f) ? g[i] : 0.f;
        d0[i] = first ? gy : 0.f;
        d1[i] = first ? 0.f : gy;
        s1[i] += gy;
        s2[i] += d0[i] * (x0[i] - mu[i]) * is[i] + d1[i] * (x1[i] - mu[i]) * is[i];
      }
    } else {
      float x[8], d[8];
      unpack8(cx0, x);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float y = fmaf(x[i], sc[i], sh[i]);
        d[i] = (y > 0.f) ? g[i] : 0.f;
        s1[i] += d[i];
        s2[i] += d[i] * (x[i] - mu[i]) * is[i];
      }
    }
  }
  // block reduction over the rows_per_block row groups, then one f64 atomic per channel per block
  __shared__ float sm1[256 * 8], sm2[256 * 8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { sm1[threadIdx.x * 8 + i] = s1[i]; sm2[threadIdx.x * 8 + i] = s2[i]; }
  __syncthreads();
  if (threadIdx.x < vpc) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float a = 0.f, b = 0.f;
      for (int r = 0; r < rows_per_block; ++r) { a += sm1[(r * vpc + threadIdx.x) * 8 + i]; b += sm2[(r * vpc + threadIdx.x) * 8 + i]; }
      atomicAdd(sums + c + i, (double)a);
      atomicAdd(sums + C + c + i, (double)b);
    }
  }
}

// pass 2a: per-channel coefficients of  dx = A*dy + B + C*x   (from dx = gamma*invstd*(dy - mean(dy) - xhat*mean(dy*xhat))),
// plus dgamma = sum(dy*xhat), dbeta = sum(dy)
// `sums` / `count` describe the batch the statistics were taken over (the GLOBAL batch under data parallelism); the gamma / beta
// gradients accumulate this rank's LOCAL sums (the flat gradient buffers are summed over ranks afterwards).
__global__ void bn_bwd_coef_kernel(const float* __restrict__ bn, const float* __restrict__ gamma, const double* __restrict__ sums,
                                   const double* __restrict__ sums_local, double count, int C, float* __restrict__ coef,
                                   float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double mu = bn[2 * C + c], is = bn[3 * C + c], g = gamma[c];
  const double m1 = sums[c] / count, m2 = sums[C + c] / count;
  coef[c] = (float)(g * is);
  coef[C + c] = (float)(-g * is * m1 + g * is * is * m2 * mu);
  coef[2 * C + c] = (float)(-g * is * is * m2);
  dbeta[c] += (float)sums_local[c];
  dgamma[c] += (float)sums_local[C + c];
}
// pass 2b: dx = A*dy + B + C*x with dy re-derived from (dout, x_pre) exactly as pass 1 derived it (the masked / routed values are
// copies of bf16 inputs, so both passes see identical numbers).  POOL: one thread per POOLED position and 8 channels, writes the
// two pre-pool positions; else elementwise (dx may alias dout).
template <bool POOL>
__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const uint4* dout, const uint4* __restrict__ x_pre,
                                                           const float* __restrict__ bn, const float* __restrict__ coef,
                                                           uint4* dx, size_t nvec_out, int C) {
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i0 >= nvec_out) return;
  const int vpc = C / 8;
  const size_t pos = i0 / vpc;
  const int cv = (int)(i0 - pos * vpc);
  const int c = cv * 8;
  float g[8], A[8], B[8], Cc[8], sc[8], sh[8];
  unpack8(POOL ? __ldg(dout + i0) : dout[i0], g);          // !POOL: dx aliases dout (same element, read before written)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float4 a4 = __ldg(reinterpret_cast<const float4*>(coef + c) + h), b4 = __ldg(reinterpret_cast<const float4*>(coef + C + c) + h),
                 c4 = __ldg(reinterpret_cast<const float4*>(coef + 2 * C + c) + h);
    const float4 s4 = __ldg(reinterpret_cast<const float4*>(bn + c) + h), h4 = __ldg(reinterpret_cast<const float4*>(bn + C + c) + h);
    A[4 * h] = a4.x; A[4 * h + 1] = a4.y; A[4 * h + 2] = a4.z; A[4 * h + 3] = a4.w;
    B[4 * h] = b4.x; B[4 * h + 1] = b4.y; B[4 * h + 2] = b4.z; B[4 * h + 3] = b4.w;
    Cc[4 * h] = c4.x; Cc[4 * h + 1] = c4.y; Cc[4 * h + 2] = c4.z; Cc[4 * h + 3] = c4.w;
    sc[4 * h] = s4.x; sc[4 * h + 1] = s4.y; sc[4 * h + 2] = s4.z; sc[4 * h + 3] = s4.w;
    sh[4 * h] = h4.x; sh[4 * h + 1] = h4.y; sh[4 * h + 2] = h4.z; sh[4 * h + 3] = h4.w;
  }
  if (POOL) {
    float x0[8], x1[8], o0[8], o1[8];
    unpack8(__ldg(x_pre + (2 * pos) * vpc + cv), x0);
    unpack8(__ldg(x_pre + (2 * pos + 1) * vpc + cv), x1);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float y0 = __bfloat162float(__float2bfloat16_rn(fmaxf(fmaf(x0[i], sc[i], sh[i]), 0.f)));
      const float y1 = __bfloat162float(__float2bfloat16_rn(fmaxf(fmaf(x1[i], sc[i], sh[i]), 0.f)));
      const bool first = (y0 >= y1);
      const float gy = ((first ? y0 : y1) > 0.f) ? g[i] : 0.f;
      o0[i] = fmaf(A[i], first ? gy : 0.f, fmaf(Cc[i], x0[i], B[i]));
      o1[i] = fmaf(A[i], first ? 0.f : gy, fmaf(Cc[i], x1[i], B[i]));
    }
    dx[(2 * pos) * vpc + cv] = pack8(o0);
    dx[(2 * pos + 1) * vpc + cv] = pack8(o1);
  } else {
    float x[8], o[8];
    unpack8(__ldg(x_pre + i0), x);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float y = fmaf(x[i], sc[i], sh[i]);
      o[i] = fmaf(A[i], (y > 0.f) ? g[i] : 0.f, fmaf(Cc[i], x[i], B[i]));
    }
    dx[i0] = pack8(o);
  }
}

// ---- un-pool + ReLU backward.  WIN = 2 (1x2 over the Wd axis, conv3_2) or 4 (2x2, conv2).
// dpool/pooled/argmax: [Npos_out..., C]; dpre: pre-pool resolution.  Geometry: pooled [N, Hp, Wp, C];
// pre-pool [N, Hp*(WIN==4?2:1), Wp*2, C].
template <int WIN>
__global__ void __launch_bounds__(256) unpool_relu_bwd_kernel(const uint4* __restrict__ dpool, const uint4* __restrict__ pooled,
                                                              const uint2* __restrict__ argmax, uint4* __restrict__ dpre,
                                                              size_t nvec_out, int Hp, int Wp, int C) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nvec_out) return;
  const int vpc = C / 8;
  const size_t pos = i / vpc;
  const int cv = (int)(i - pos * vpc);
  const int wp = (int)(pos % Wp);
  const size_t nh = pos / Wp;               // n*Hp + hp
  float g[8], y[8];
  unpack8(__ldg(dpool + i), g);
  unpack8(__ldg(pooled + i), y);
  const uint2 am = __ldg(argmax + i);
  uint32_t idx[8] = {am.x & 255u, (am.x >> 8) & 255u, (am.x >> 16) & 255u, am.x >> 24,
                     am.y & 255u, (am.y >> 8) & 255u, (am.y >> 16) & 255u, am.y >> 24};
#pragma unroll
  for (int k = 0; k < 8; ++k) g[k] = (y[k] > 0.f) ? g[k] : 0.f;
#pragma unroll
  for (int wdx = 0; wdx < WIN; ++wdx) {
    float o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = (idx[k] == (uint32_t)wdx) ? g[k] : 0.f;
    size_t dst_pos;
    if (WIN == 2) dst_pos = nh * (2 * Wp) + 2 * wp + wdx;
    else dst_pos = (nh * 2 + (wdx >> 1)) * (size_t)(2 * Wp) + 2 * wp + (wdx & 1);
    dpre[dst_pos * vpc + cv] = pack8(o);
  }
}

// ---- weight re-layouts for the backward GEMMs (bf16, K-major B operands) ---------------------------------------
// data-gradient of a 3x3 SAME conv == 3x3 SAME conv of dY with the spatially flipped, in/out-swapped kernel:
//   Bd[ci][(r',s',co)] = W[2-r'][2-s'][ci][co]       (W is HWIO)
__global__ void dgrad_weight_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ bd, int Cin, int Cout) {
  const size_t total = (size_t)Cin * 9 * Cout;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int co = (int)(i % Cout);
    const size_t t = i / Cout;
    const int tap = (int)(t % 9);
    const int ci = (int)(t / 9);
    const int r = tap / 3, s = tap % 3;
    bd[i] = __float2bfloat16_rn(w[(((size_t)(2 - r) * 3 + (2 - s)) * Cin + ci) * Cout + co]);
  }
}
// conv5 (2x2 VALID over [N,H,2,512]) data gradient: Bd[(w,ci)][(r,co)] = W[r][w][ci][co]
__global__ void conv5_dgrad_weight_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ bd) {
  const size_t total = (size_t)1024 * 1024;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int co = (int)(i & 511);
    const int r = (int)((i >> 9) & 1);
    const int wc = (int)(i >> 10);                 // (w, ci) in 0..1023
    bd[i] = __float2bfloat16_rn(w[((size_t)r * 1024 + wc) * 512 + co]);
  }
}
// LSTM: rows of the TF matrix [768,1024] with gate columns permuted (upc = LSTM_GATE_UNITS), both directions.
//   bxb[x][dir*1024 + p] (x < 512, dx GEMM)      bhb[dir*256 + u][p] (recurrent backward GEMM)
__global__ void lstm_bwd_weight_kernel(const float* __restrict__ w_fw, const float* __restrict__ w_bw,
                                       __nv_bfloat16* __restrict__ bxb, __nv_bfloat16* __restrict__ bhb, int upc) {
  const size_t total = (size_t)2 * 768 * 1024;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int p = (int)(i & 1023);
    const int row = (int)((i >> 10) % 768);
    const int dir = (int)(i / ((size_t)768 * 1024));
    const int g = (p % (4 * upc)) / upc, u = (p / (4 * upc)) * upc + p % upc;
    const float v = (dir ? w_bw : w_fw)[(size_t)row * 1024 + g * 256 + u];
    if (row < 512) bxb[(size_t)row * 2048 + dir * 1024 + p] = __float2bfloat16_rn(v);
    else bhb[((size_t)dir * 256 + (row - 512)) * 1024 + p] = __float2bfloat16_rn(v);
  }
}
__global__ void cast_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    dst[i] = __float2bfloat16_rn(src[i]);
}

// ---- optimizer: L2-term gradient + global norm, then clip + Adam / Momentum / RMSProp (TF formulas, lib/lstm/train.py:73-83)
__global__ void __launch_bounds__(256) grad_finish_kernel(float* __restrict__ grads, const float* __restrict__ params,
                                                          WdSegs segs, float wd, long long total, double* __restrict__ sumsq) {
  double acc = 0.0;
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < total; i += (long long)gridDim.x * blockDim.x * 4) {
    float4 g = *reinterpret_cast<float4*>(grads + i);
    bool reg = false;
#pragma unroll
    for (int s = 0; s < 8; ++s) reg = reg || (s < segs.n && i >= segs.off[s] && i < segs.off[s] + segs.cnt[s]);
    if (reg && wd > 0.f) {
      const float4 w = __ldg(reinterpret_cast<const float4*>(params + i));
      g.x = fmaf(wd, w.x, g.x); g.y = fmaf(wd, w.y, g.y); g.z = fmaf(wd, w.z, g.z); g.w = fmaf(wd, w.w, g.w);
      *reinterpret_cast<float4*>(grads + i) = g;
    }
    acc += (double)g.x * g.x + (double)g.y * g.y + (double)g.z * g.z + (double)g.w * g.w;
  }
  __shared__ double red[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int i = 0; i < 8; ++i) t += red[i];
    atomicAdd(sumsq, t);
  }
}
// Factor applied to every raw gradient element: the averaging factor times tf.clip_by_global_norm's clip / max(norm, clip),
// where the global norm of the (already averaged) gradient is sqrt(sumsq) * grad_mul.  clip <= 0 disables clipping.
__device__ __forceinline__ float clip_scale(const double* __restrict__ sumsq, float grad_mul, float clip) {
  const float gn = (float)sqrt(*sumsq) * grad_mul;
  return grad_mul * (clip > 0.f ? clip / fmaxf(gn, clip) : 1.f);
}
__global__ void __launch_bounds__(256) clip_adam_kernel(float* __restrict__ params, const float* __restrict__ grads,
                                                        float* __restrict__ m, float* __restrict__ v,
                                                        const double* __restrict__ sumsq, float grad_mul, float clip, float lr_t,
                                                        float b1, float b2, float eps, long long total) {
  const float scale = clip_scale(sumsq, grad_mul, clip);
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < total; i += (long long)gridDim.x * blockDim.x * 4) {
    const float4 g4 = __ldg(reinterpret_cast<const float4*>(grads + i));
    float4 p4 = *reinterpret_cast<float4*>(params + i), m4 = *reinterpret_cast<float4*>(m + i), v4 = *reinterpret_cast<float4*>(v + i);
    float* pp = &p4.x; float* mm = &m4.x; float* vv = &v4.x; const float* gg = &g4.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float g = gg[k] * scale;
      mm[k] = b1 * mm[k] + (1.f - b1) * g;
      vv[k] = b2 * vv[k] + (1.f - b2) * g * g;
      pp[k] -= lr_t * mm[k] / (sqrtf(vv[k]) + eps);
    }
    *reinterpret_cast<float4*>(params + i) = p4;
    *reinterpret_cast<float4*>(m + i) = m4;
    *reinterpret_cast<float4*>(v + i) = v4;
  }
}
// TF MomentumOptimizer (use_nesterov=False, ApplyMomentum): accum = accum*momentum + g; var -= lr*accum.  lr multiplies the whole
// accumulator when it is applied, so a decayed lr shrinks the step taken from the accumulated velocity at once.
__global__ void __launch_bounds__(256) clip_momentum_kernel(float* __restrict__ params, const float* __restrict__ grads,
                                                            float* __restrict__ accum, const double* __restrict__ sumsq, float grad_mul,
                                                            float clip, float lr, float momentum, long long total) {
  const float scale = clip_scale(sumsq, grad_mul, clip);
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < total; i += (long long)gridDim.x * blockDim.x * 4) {
    const float4 g4 = __ldg(reinterpret_cast<const float4*>(grads + i));
    float4 p4 = *reinterpret_cast<float4*>(params + i), a4 = *reinterpret_cast<float4*>(accum + i);
    float* pp = &p4.x; float* aa = &a4.x; const float* gg = &g4.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float g = gg[k] * scale;
      aa[k] = aa[k] * momentum + g;
      pp[k] -= lr * aa[k];
    }
    *reinterpret_cast<float4*>(params + i) = p4;
    *reinterpret_cast<float4*>(accum + i) = a4;
  }
}
// TF RMSPropOptimizer (centered=False, ApplyRMSProp): ms += (g*g - ms)*(1 - decay); mom = mom*momentum + lr*g/sqrt(ms + eps);
// var -= mom.  eps sits inside the square root; TF starts ms at 1.0 (the caller initialises it).
__global__ void __launch_bounds__(256) clip_rmsprop_kernel(float* __restrict__ params, const float* __restrict__ grads,
                                                           float* __restrict__ mom, float* __restrict__ ms,
                                                           const double* __restrict__ sumsq, float grad_mul, float clip, float lr,
                                                           float decay, float momentum, float eps, long long total) {
  const float scale = clip_scale(sumsq, grad_mul, clip);
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < total; i += (long long)gridDim.x * blockDim.x * 4) {
    const float4 g4 = __ldg(reinterpret_cast<const float4*>(grads + i));
    float4 p4 = *reinterpret_cast<float4*>(params + i), m4 = *reinterpret_cast<float4*>(mom + i), s4 = *reinterpret_cast<float4*>(ms + i);
    float* pp = &p4.x; float* mm = &m4.x; float* ss = &s4.x; const float* gg = &g4.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float g = gg[k] * scale;
      ss[k] += (g * g - ss[k]) * (1.f - decay);
      mm[k] = mm[k] * momentum + lr * g / sqrtf(ss[k] + eps);
      pp[k] -= mm[k];
    }
    *reinterpret_cast<float4*>(params + i) = p4;
    *reinterpret_cast<float4*>(mom + i) = m4;
    *reinterpret_cast<float4*>(ms + i) = s4;
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------------ launchers
#define LAUNCH_CHECK() CUDA_TRY(cudaGetLastError()); return CRNN_OK

// SM count of the current device: the grid-stride kernels below launch a few CTAs per SM
static int device_sms() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
  if (cached[dev] <= 0) cudaDeviceGetAttribute(&cached[dev], cudaDevAttrMultiProcessorCount, dev);
  return cached[dev] > 0 ? cached[dev] : 1;
}

int launch_dlogits_rows(const float* dlogits, __nv_bfloat16* rows, float* dbias, int T, int N, int H, cudaStream_t st) {
  dlogits_rows_kernel<<<4 * device_sms(), 256, 0, st>>>(dlogits, rows, dbias, T, N, H);
  LAUNCH_CHECK();
}
int launch_colsum_bf16(const __nv_bfloat16* src, long long R, int C, float* out, bool lstm_gates, long long dir_stride, cudaStream_t st) {
  dim3 grid(2 * device_sms(), (C + 255) / 256);
  colsum_bf16_kernel<<<grid, 256, 0, st>>>(src, nullptr, R, C, 0, out, lstm_gates ? LSTM_GATE_UNITS : 0, dir_stride);
  LAUNCH_CHECK();
}
// out[c] += sum over rows of src[r][c] where mask[r][c] > 0.  Narrow tensors (C = 128) are read as a [R/2, 256] view so that
// every lane of the 256-column block works.
int launch_colsum_masked_bf16(const __nv_bfloat16* src, const __nv_bfloat16* mask, long long R, int C, float* out, cudaStream_t st) {
  int Cv = C, Cmod = 0;
  long long Rv = R;
  if (C < 256 && 256 % C == 0 && R % (256 / C) == 0) { Cv = 256; Cmod = C; Rv = R / (256 / C); }
  dim3 grid(2 * device_sms(), (Cv + 255) / 256);
  colsum_bf16_kernel<<<grid, 256, 0, st>>>(src, mask, Rv, Cv, Cmod, out, 0, 0);
  LAUNCH_CHECK();
}
int launch_bn_bwd_reduce(const __nv_bfloat16* dout, const __nv_bfloat16* x_pre, const float* bn, double* sums, size_t out_positions, int C,
                         cudaStream_t st) {
  bn_bwd_reduce_kernel<true><<<4 * device_sms(), 256, 0, st>>>((const uint4*)dout, (const uint4*)x_pre, nullptr, bn, sums, out_positions, C);
  LAUNCH_CHECK();
}
// dx = BN/ReLU(/pool) backward of dout; out_positions = positions of dout (pooled positions when pool); dx may alias dout when !pool
int launch_bn_bwd_apply(bool pool, const __nv_bfloat16* dout, const __nv_bfloat16* x_pre, __nv_bfloat16* dx, const float* bn,
                        const float* gamma, const double* sums, const double* sums_local, double count, size_t out_positions, int C,
                        float* coef, float* dgamma, float* dbeta, cudaStream_t st) {
  const size_t nvec = out_positions * C / 8;
  bn_bwd_coef_kernel<<<(C + 127) / 128, 128, 0, st>>>(bn, gamma, sums, sums_local, count, C, coef, dgamma, dbeta);
  CUDA_TRY(cudaGetLastError());
  if (pool) bn_bwd_apply_kernel<true><<<(unsigned)((nvec + 255) / 256), 256, 0, st>>>((const uint4*)dout, (const uint4*)x_pre, bn, coef, (uint4*)dx, nvec, C);
  else bn_bwd_apply_kernel<false><<<(unsigned)((nvec + 255) / 256), 256, 0, st>>>((const uint4*)dout, (const uint4*)x_pre, bn, coef, (uint4*)dx, nvec, C);
  LAUNCH_CHECK();
}
int launch_unpool_relu_bwd(int win, const __nv_bfloat16* dpool, const __nv_bfloat16* pooled, const uint8_t* argmax,
                           __nv_bfloat16* dpre, size_t out_positions, int Hp, int Wp, int C, cudaStream_t st) {
  const size_t nvec = out_positions * C / 8;
  const unsigned grid = (unsigned)((nvec + 255) / 256);
  if (win == 2) unpool_relu_bwd_kernel<2><<<grid, 256, 0, st>>>((const uint4*)dpool, (const uint4*)pooled, (const uint2*)argmax, (uint4*)dpre, nvec, Hp, Wp, C);
  else unpool_relu_bwd_kernel<4><<<grid, 256, 0, st>>>((const uint4*)dpool, (const uint4*)pooled, (const uint2*)argmax, (uint4*)dpre, nvec, Hp, Wp, C);
  LAUNCH_CHECK();
}
int launch_dgrad_weight(const float* w, __nv_bfloat16* bd, int Cin, int Cout, cudaStream_t st) {
  dgrad_weight_kernel<<<4 * device_sms(), 256, 0, st>>>(w, bd, Cin, Cout);
  LAUNCH_CHECK();
}
int launch_conv5_dgrad_weight(const float* w, __nv_bfloat16* bd, cudaStream_t st) {
  conv5_dgrad_weight_kernel<<<4 * device_sms(), 256, 0, st>>>(w, bd);
  LAUNCH_CHECK();
}
int launch_lstm_bwd_weight(const float* w_fw, const float* w_bw, __nv_bfloat16* bxb, __nv_bfloat16* bhb, cudaStream_t st) {
  lstm_bwd_weight_kernel<<<4 * device_sms(), 256, 0, st>>>(w_fw, w_bw, bxb, bhb, LSTM_GATE_UNITS);
  LAUNCH_CHECK();
}
int launch_cast_bf16(const float* src, __nv_bfloat16* dst, size_t n, cudaStream_t st) {
  cast_bf16_kernel<<<device_sms(), 256, 0, st>>>(src, dst, n);
  LAUNCH_CHECK();
}
int launch_grad_finish(float* grads, const float* params, const WdSegs& segs, float wd, long long total, double* sumsq, cudaStream_t st) {
  CUDA_TRY(cudaMemsetAsync(sumsq, 0, sizeof(double), st));
  grad_finish_kernel<<<4 * device_sms(), 256, 0, st>>>(grads, params, segs, wd, total, sumsq);
  LAUNCH_CHECK();
}
int launch_clip_adam(float* params, const float* grads, float* m, float* v, const double* sumsq, float grad_mul, float clip, float lr_t,
                     float b1, float b2, float eps, long long total, cudaStream_t st) {
  clip_adam_kernel<<<4 * device_sms(), 256, 0, st>>>(params, grads, m, v, sumsq, grad_mul, clip, lr_t, b1, b2, eps, total);
  LAUNCH_CHECK();
}
int launch_clip_momentum(float* params, const float* grads, float* accum, const double* sumsq, float grad_mul, float clip, float lr,
                         float momentum, long long total, cudaStream_t st) {
  clip_momentum_kernel<<<4 * device_sms(), 256, 0, st>>>(params, grads, accum, sumsq, grad_mul, clip, lr, momentum, total);
  LAUNCH_CHECK();
}
int launch_clip_rmsprop(float* params, const float* grads, float* mom, float* ms, const double* sumsq, float grad_mul, float clip,
                        float lr, float decay, float momentum, float eps, long long total, cudaStream_t st) {
  clip_rmsprop_kernel<<<4 * device_sms(), 256, 0, st>>>(params, grads, mom, ms, sumsq, grad_mul, clip, lr, decay, momentum, eps, total);
  LAUNCH_CHECK();
}
