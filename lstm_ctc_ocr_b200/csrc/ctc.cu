// CTC loss (+ gradient) and greedy decode for C = 64 classes, sm_90a.
//
// Replaces warpctc_tensorflow.ctc at lib/networks/network.py:653-654 and the decode at
// lib/networks/network.py:656-657 (+ zero stripping, lib/lstm/utils/training.py:32).
//
// Two kernels, same arithmetic (log2-space recursions, softmax with max subtraction inside):
//
// ctc_fast_kernel (S = 2L+1 <= 32, the captcha/text-line case): one 64-thread CTA per utterance, 8 CTAs per SM.
//   load     every thread pulls its own frames' 256-B logit rows into shared memory with 1-D bulk copies (no LSU work)
//   phase 0  thread = frame: row max, p = 2^(x-m) written back in place, normaliser, the L+1 emission scores of the frame
//   phase 1  the alpha and the (state-reversed) beta recursion are the SAME instruction stream -- value from lane-1 / lane-2
//            via warp shuffles -- so for S <= 16 they share one warp (lanes 0-15 alpha, 16-31 beta); for S <= 32 warp 0 / warp 1
//   phase 2  thread = frame: row <- scale*p/sum, minus the state posteriors scattered into the thread's own row (no
//            atomics), then one 256-B bulk store of the row to the gradient
//
// ctc_loss_kernel<KS> (S <= 32*KS, generic): one CTA (4 warps) per utterance; warps 0/1 run the two recursions, all 4 share
// the frame-parallel phases.
//   phase 0  both warps, rows interleaved: log2-softmax normaliser per frame and the S <= 32*KS
//            emission scores e[t][s] = log2 y_t(l'_s), kept in shared memory (HBM read #1, coalesced 256 B rows)
//   phase 1  warp 0 runs the alpha recursion forward while warp 1 runs the beta recursion backward --
//            the two 63-step dependency chains overlap; each step is a warp-shuffle scan over the states
//            (lane owns KS consecutive states, neighbours via __shfl_up/__shfl_down), all in log2 space
//   phase 2  both warps, rows interleaved: re-read the logits row (L2 hit), y = softmax, per-class
//            sum of alpha*beta/y via shared-memory accumulators, write grad row (HBM write, coalesced)
// ctc_long_kernel (max_label_len <= 639, any T): the caller's workspace holds the log-softmax and alpha tables that do not
//   fit in shared memory; it runs where the kernels above cannot (see its comment below).
// No tensor cores: the dynamic program is a scan, not a contraction.
#include "common.cuh"
#include <cuda.h>
#include <limits.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace {

constexpr int CTC_C = 64;
constexpr int CTC_WARPS = 4;                 // phases 0/2 are parallel over frames: 4 warps x 16 rows covers T <= 64 in one batch
constexpr int CTC_THREADS = 32 * CTC_WARPS;
constexpr int CTC_RB = 16;                   // rows per warp per batch: all 16 loads are issued before any use (MLP)
constexpr int CTC_RG = 4;                    // rows reduced in lockstep (ILP) within a batch
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;
#define NEG_INF (-INFINITY)

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// Two adjacent floats of a logit / gradient row.  The generic kernel also takes pointers that are only 4-byte aligned
// (every misaligned call is routed to it); there the pair is moved as two scalars, with the same values.
__device__ __forceinline__ float2 ld_pair(const float* p, bool vec) {
  return vec ? __ldg(reinterpret_cast<const float2*>(p)) : make_float2(__ldg(p), __ldg(p + 1));
}
__device__ __forceinline__ void st_pair(float* p, float2 v, bool vec) {
  if (vec) {
    *reinterpret_cast<float2*>(p) = v;
  } else {
    p[0] = v.x;
    p[1] = v.y;
  }
}
// 3-input maximum (exact: the order of two-operand maxima does not change the result)
__device__ __forceinline__ float max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
// log2(2^a + 2^b + 2^c) with -inf handling
__device__ __forceinline__ float lse3(float a, float b, float c) {
  float m = fmaxf(a, fmaxf(b, c));
  if (m == NEG_INF) return NEG_INF;
  return m + ptx::lg2(ptx::ex2(a - m) + ptx::ex2(b - m) + ptx::ex2(c - m));
}

template <int KS>
__global__ void __launch_bounds__(CTC_THREADS, 8) ctc_loss_kernel(const float* __restrict__ logits, float* __restrict__ grad,
                                                      const int* __restrict__ flat_labels,
                                                      const int* __restrict__ label_len,
                                                      const int* __restrict__ input_len, int T, int N, int blank,
                                                      float grad_scale, float* __restrict__ costs) {
  constexpr int SP = 32 * KS;  // padded state count
  extern __shared__ float sm[];
  float* s_lse = sm;                    // [T]
  float* s_e = s_lse + T;               // [T][SP]
  float* s_alpha = s_e + (size_t)T * SP;
  float* s_beta = s_alpha + (size_t)T * SP;
  float* s_acc = s_beta + (size_t)T * SP;   // [4 warps][4 rows][64]
  __shared__ int s_off;
  __shared__ int s_ext[SP];
  __shared__ int s_repeats;
  __shared__ int s_bad;

  const int n = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int L = label_len[n];
  int Tn = input_len[n];
  Tn = max(0, min(Tn, T));
  const int S = 2 * L + 1;
  const bool lvec = (reinterpret_cast<uintptr_t>(logits) & 7) == 0, gvec = (reinterpret_cast<uintptr_t>(grad) & 7) == 0;

  // label offset = sum(label_len[0..n))
  if (warp == 0) {
    int acc = 0;
    for (int i = lane; i < n; i += 32) acc += label_len[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) s_off = acc;
  }
  __syncthreads();
  bool too_long = (S > SP) || (L < 0);
  if (threadIdx.x == 0) { s_repeats = 0; s_bad = 0; }
  __syncthreads();
  if (!too_long) {
    int rep = 0, bad = 0;
    for (int s = threadIdx.x; s < SP; s += CTC_THREADS) {
      int v = blank;
      if (s < S && (s & 1)) {
        v = flat_labels[s_off + (s >> 1)];
        // a label id outside [0,C) or equal to the blank would index the 64-class rows out of bounds / alias the blank
        // states: the sample is rejected (cost NaN, zero gradient) and the id is never used as an index
        if (v < 0 || v >= CTC_C || v == blank) { bad = 1; v = blank; }
        if (s >= 3 && v == flat_labels[s_off + (s >> 1) - 1]) rep++;
      }
      s_ext[s] = v;
    }
    if (rep) atomicAdd(&s_repeats, rep);
    if (bad) atomicOr(&s_bad, 1);
  }
  __syncthreads();
  too_long = too_long || (s_bad != 0);

  const bool feasible = !too_long && Tn > 0 && (L + s_repeats <= Tn);
  if (!feasible) {
    if (threadIdx.x == 0) costs[n] = too_long ? __int_as_float(0x7fc00000) : 0.0f;
    if (grad != nullptr) {
      for (int t = warp; t < T; t += CTC_WARPS)
        st_pair(grad + ((size_t)t * N + n) * CTC_C + 2 * lane, make_float2(0.f, 0.f), gvec);
    }
    return;
  }

  // ---------------- phase 0: normalisers + emission gather ----------------
  int cls[KS];
#pragma unroll
  for (int k = 0; k < KS; ++k) cls[k] = s_ext[lane * KS + k];
  for (int t0 = warp; t0 < Tn; t0 += CTC_WARPS * CTC_RB) {
    float2 xr[CTC_RB];
#pragma unroll
    for (int u = 0; u < CTC_RB; ++u) {
      const int t = t0 + CTC_WARPS * u;
      xr[u] = (t < Tn) ? ld_pair(logits + ((size_t)t * N + n) * CTC_C + 2 * lane, lvec) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int g = 0; g < CTC_RB; g += CTC_RG) {
      if (t0 + CTC_WARPS * g >= Tn) break;               // warp-uniform
      float x0[CTC_RG], x1[CTC_RG], m[CTC_RG], sum[CTC_RG];
#pragma unroll
      for (int u = 0; u < CTC_RG; ++u) {
        x0[u] = xr[g + u].x * LOG2E; x1[u] = xr[g + u].y * LOG2E;
        m[u] = fmaxf(x0[u], x1[u]);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int u = 0; u < CTC_RG; ++u) m[u] = fmaxf(m[u], __shfl_xor_sync(0xffffffffu, m[u], o));
#pragma unroll
      for (int u = 0; u < CTC_RG; ++u) sum[u] = ptx::ex2(x0[u] - m[u]) + ptx::ex2(x1[u] - m[u]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int u = 0; u < CTC_RG; ++u) sum[u] += __shfl_xor_sync(0xffffffffu, sum[u], o);
#pragma unroll
      for (int u = 0; u < CTC_RG; ++u) {
        const int t = t0 + CTC_WARPS * (g + u);
        const float lse = m[u] + ptx::lg2(sum[u]);
#pragma unroll
        for (int k = 0; k < KS; ++k) {
          const int c = cls[k];
          const float v0 = __shfl_sync(0xffffffffu, x0[u], c >> 1);
          const float v1 = __shfl_sync(0xffffffffu, x1[u], c >> 1);
          if (t < Tn) s_e[(size_t)t * SP + lane * KS + k] = ((c & 1) ? v1 : v0) - lse;
        }
        if (lane == 0 && t < Tn) s_lse[t] = lse;
      }
    }
  }
  __syncthreads();

  // ---------------- phase 1: alpha (warp 0) || beta (warp 1) ----------------
  {
    // skip transition allowed into state s from s-2 (alpha) / from s into s+2 (beta)
    bool skip_in[KS], skip_out[KS];
#pragma unroll
    for (int k = 0; k < KS; ++k) {
      int s = lane * KS + k;
      skip_in[k] = (s >= 2) && (s < S) && (s_ext[s] != blank) && (s_ext[s] != s_ext[s - 2]);
      skip_out[k] = (s + 2 < S) && (s_ext[s + 2] != blank) && (s_ext[s + 2] != s_ext[s]);
    }
    float a[KS];
    if (warp >= 2) {
      // idle during the two recursions (frame-parallel phases only)
    } else if (warp == 0) {
#pragma unroll
      for (int k = 0; k < KS; ++k) {
        int s = lane * KS + k;
        a[k] = (s < 2 && s < S) ? s_e[s] : NEG_INF;
        s_alpha[s] = a[k];
      }
      for (int t = 1; t < Tn; ++t) {
        float up1 = __shfl_up_sync(0xffffffffu, a[KS - 1], 1);
        float up2 = (KS >= 2) ? __shfl_up_sync(0xffffffffu, a[(KS >= 2) ? KS - 2 : 0], 1)
                              : __shfl_up_sync(0xffffffffu, a[0], 2);
        if (lane == 0) { up1 = NEG_INF; up2 = NEG_INF; }
        if (KS == 1 && lane == 1) up2 = NEG_INF;
        float nw[KS];
#pragma unroll
        for (int k = 0; k < KS; ++k) {
          float p1 = (k >= 1) ? a[(k >= 1) ? k - 1 : 0] : up1;
          float p2 = (k >= 2) ? a[(k >= 2) ? k - 2 : 0] : ((k == 1) ? up1 : up2);
          if (!skip_in[k]) p2 = NEG_INF;
          int s = lane * KS + k;
          float v = lse3(a[k], p1, p2) + s_e[(size_t)t * SP + s];
          nw[k] = (s < S) ? v : NEG_INF;
        }
#pragma unroll
        for (int k = 0; k < KS; ++k) {
          a[k] = nw[k];
          s_alpha[(size_t)t * SP + lane * KS + k] = a[k];
        }
      }
    } else {
#pragma unroll
      for (int k = 0; k < KS; ++k) {
        int s = lane * KS + k;
        a[k] = (s < S && s >= S - 2) ? s_e[(size_t)(Tn - 1) * SP + s] : NEG_INF;
        s_beta[(size_t)(Tn - 1) * SP + s] = a[k];
      }
      for (int t = Tn - 2; t >= 0; --t) {
        float dn1 = __shfl_down_sync(0xffffffffu, a[0], 1);
        float dn2 = (KS >= 2) ? __shfl_down_sync(0xffffffffu, a[(KS >= 2) ? 1 : 0], 1)
                              : __shfl_down_sync(0xffffffffu, a[0], 2);
        if (lane == 31) { dn1 = NEG_INF; dn2 = NEG_INF; }
        if (KS == 1 && lane == 30) dn2 = NEG_INF;
        float nw[KS];
#pragma unroll
        for (int k = 0; k < KS; ++k) {
          float p1 = (k + 1 < KS) ? a[(k + 1 < KS) ? k + 1 : 0] : dn1;
          // state s+2: own register, else neighbour's first (dn1) or second / lane+2's (dn2)
          float p2 = (k + 2 < KS) ? a[(k + 2 < KS) ? k + 2 : 0] : ((k + 1 < KS) ? dn1 : dn2);
          if (!skip_out[k]) p2 = NEG_INF;
          int s = lane * KS + k;
          float v = lse3(a[k], p1, p2) + s_e[(size_t)t * SP + s];
          nw[k] = (s < S) ? v : NEG_INF;
        }
#pragma unroll
        for (int k = 0; k < KS; ++k) {
          a[k] = nw[k];
          s_beta[(size_t)t * SP + lane * KS + k] = a[k];
        }
      }
    }
  }
  __syncthreads();

  // log2-likelihood from the last alpha row
  const float aS1 = s_alpha[(size_t)(Tn - 1) * SP + (S - 1)];
  const float aS2 = (S >= 2) ? s_alpha[(size_t)(Tn - 1) * SP + (S - 2)] : NEG_INF;
  const float ll2 = lse3(aS1, aS2, NEG_INF);
  if (threadIdx.x == 0) costs[n] = -ll2 * LN2;
  if (grad == nullptr) return;

  // ---------------- phase 2: gradient rows ----------------
  float* acc = s_acc + warp * CTC_RG * CTC_C;         // [CTC_RG rows][64] per warp
  for (int t0 = warp; t0 < T; t0 += CTC_WARPS * CTC_RB) {
    float2 xr[CTC_RB];
#pragma unroll
    for (int u = 0; u < CTC_RB; ++u) {
      const int t = t0 + CTC_WARPS * u;
      xr[u] = ((t < Tn) && (ll2 != NEG_INF)) ? ld_pair(logits + ((size_t)t * N + n) * CTC_C + 2 * lane, lvec)
                                             : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int g = 0; g < CTC_RB; g += CTC_RG) {
      if (t0 + CTC_WARPS * g >= T) break;                 // warp-uniform
      bool live[CTC_RG];
#pragma unroll
      for (int u = 0; u < CTC_RG; ++u) {
        const int t = t0 + CTC_WARPS * (g + u);
        live[u] = (t < Tn) && (ll2 != NEG_INF);
        acc[u * CTC_C + 2 * lane] = 0.f;
        acc[u * CTC_C + 2 * lane + 1] = 0.f;
      }
      __syncwarp();
      float blank_sum[CTC_RG];
#pragma unroll
      for (int u = 0; u < CTC_RG; ++u) {
        const int t = t0 + CTC_WARPS * (g + u);
        blank_sum[u] = 0.f;
        if (live[u]) {
#pragma unroll
          for (int k = 0; k < KS; ++k) {
            const int st = lane * KS + k;
            if (st < S) {
              const size_t i = (size_t)t * SP + st;
              const float w = ptx::ex2(s_alpha[i] + s_beta[i] - s_e[i] - ll2);   // alpha*beta / y / p(l|x)
              if (st & 1) atomicAdd(&acc[u * CTC_C + cls[k]], w);
              else blank_sum[u] += w;
            }
          }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int u = 0; u < CTC_RG; ++u) blank_sum[u] += __shfl_xor_sync(0xffffffffu, blank_sum[u], o);
      if (lane == 0) {
#pragma unroll
        for (int u = 0; u < CTC_RG; ++u) atomicAdd(&acc[u * CTC_C + blank], blank_sum[u]);
      }
      __syncwarp();
#pragma unroll
      for (int u = 0; u < CTC_RG; ++u) {
        const int t = t0 + CTC_WARPS * (g + u);
        if (t >= T) continue;
        float* gp = grad + ((size_t)t * N + n) * CTC_C + 2 * lane;
        if (!live[u]) {
          st_pair(gp, make_float2(0.f, 0.f), gvec);
        } else {
          const float lse = s_lse[t];
          const float y0 = ptx::ex2(xr[g + u].x * LOG2E - lse), y1 = ptx::ex2(xr[g + u].y * LOG2E - lse);
          st_pair(gp, make_float2(grad_scale * (y0 - acc[u * CTC_C + 2 * lane]), grad_scale * (y1 - acc[u * CTC_C + 2 * lane + 1])),
                  gvec);
        }
      }
      __syncwarp();
    }
  }
}


// ---------------------------------------------------------------------------------------------------------------------------
// Phase 1 of the S <= 32 kernels, alternative ("me" = mantissa/exponent, CRNN_CTC_RECUR=me).  The alpha/beta chain (62 dependent
// steps at T = 63) is the longest part of the kernel: every step of the log2-space recursion is SHFL -> FMNMX3 -> FADD -> MUFU.EX2 -> FADD
// -> FADD -> MUFU.LG2 -> FADD.  Here a state is carried as a PAIR
// (m in [1,2) or 0, integer exponent e), value m * 2^e: the sum of the three predecessors is three exact power-of-two scalings
// (integer shifts into the exponent field) and two FADDs, the emission is a multiplication by (ym, ye) -- split off the log2
// emission ONE STEP AHEAD, so its EX2 is off the chain --, renormalisation is integer arithmetic on the exponent field.  No
// transcendental on the dependency chain, and -- unlike a linear-space recursion with a shared per-frame scale -- no loss of
// range: the exponent is a 32-bit integer, so a state 2^-5000 below its neighbour is still carried (the log-space kernels' and
// warp-ctc's behaviour on confidently-wrong frames).  What is stored per (t, s) is still log2(alpha) = lg2(m) + e (the LG2 is
// off the chain), so phases 0 and 2 are unchanged.
// The pair arithmetic needs ~3x the dependent integer/select instructions per step, and with one or two warps per scheduler the
// chain is bound by instruction latency, not by the MUFU pipe, so this is not the faster option.  Kept as the high-accuracy option (costs agree with the fp64 oracle to ~1e-8 relative instead of ~1e-5).
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int ME_EMIN = -(1 << 28);

__device__ __forceinline__ void me_split(float z, float& ym, int& ye) {
  if (!(z > -100000.f)) { ym = 0.f; ye = 0; return; }          // log2 y below -1e5 (or NaN/-inf): probability zero
  const float fl = floorf(z);
  ym = ptx::ex2(z - fl);
  ye = (int)fl;
}
__device__ __forceinline__ float me_pow2(int d) {               // 2^d for d <= 0; 0 beyond f32 resolution of the larger addend
  return d < -64 ? 0.f : __int_as_float((d + 127) << 23);
}

__device__ __forceinline__ void ctc_recursion_me(float* s_alpha, float* s_beta, const float* s_el, const float* s_eb, const int* s_ext,
                                                 int AS, int ES, int S, int Tn, int blank, int warp, int lane) {
  const bool packed = (S <= 16);
  if (warp >= (packed ? 1 : 2)) return;
  const int W = packed ? 16 : 32;
  const int half = packed ? (lane >> 4) : warp;            // 0 = alpha, 1 = beta (state order reversed)
  const int j = packed ? (lane & 15) : lane;
  const bool valid = j < S;
  const int s = valid ? (half ? S - 1 - j : j) : 0;
  bool ok2;
  if (half == 0) ok2 = valid && (s >= 2) && (s_ext[s] != blank) && (s_ext[s] != s_ext[s - 2]);
  else           ok2 = valid && (s + 2 < S) && (s_ext[s + 2] != blank) && (s_ext[s + 2] != s_ext[s]);
  const bool ok1 = valid && j >= 1;
  const int seg = lane & ~(W - 1);
  const int src1 = seg | ((j - 1) & (W - 1)), src2 = seg | ((j - 2) & (W - 1));
  float* buf = (half ? s_beta : s_alpha) + s;
  const float* ep = (s & 1) ? (s_el + (s >> 1)) : s_eb;
  const int estride = (s & 1) ? ES : 1;
  const int dt = half ? -1 : 1;
  int t = half ? Tn - 1 : 0;
  float m, ymn = 0.f;
  int e, yen = 0;
  {
    float ym; int ye;
    me_split(ep[(size_t)t * estride], ym, ye);
    const bool live = valid && j < 2 && ym > 0.f;
    m = live ? ym : 0.f;
    e = live ? ye : ME_EMIN;
    if (valid) buf[(size_t)t * AS] = live ? ptx::lg2(m) + (float)e : NEG_INF;
  }
  if (Tn > 1) me_split(ep[(size_t)(t + dt) * estride], ymn, yen);
  for (int step = 1; step < Tn; ++step) {
    t += dt;
    const float ym = ymn;
    const int ye = yen;
    if (step + 1 < Tn) me_split(ep[(size_t)(t + dt) * estride], ymn, yen);      // next frame's emission: off the chain
    float m1 = __shfl_sync(0xffffffffu, m, src1);
    int e1 = __shfl_sync(0xffffffffu, e, src1);
    float m2 = __shfl_sync(0xffffffffu, m, src2);
    int e2 = __shfl_sync(0xffffffffu, e, src2);
    if (!ok1) { m1 = 0.f; e1 = ME_EMIN; }
    if (!ok2) { m2 = 0.f; e2 = ME_EMIN; }
    const int emax = max(e, max(e1, e2));
    const float sum = m * me_pow2(e - emax) + (m1 * me_pow2(e1 - emax) + m2 * me_pow2(e2 - emax));
    const float pr = sum * ym;                                        // [1, 12) or 0
    const uint32_t pb = __float_as_uint(pr);
    const int k = (int)(pb >> 23) - 127;
    const bool live = valid && pr > 0.f;
    m = live ? __uint_as_float(pb - ((uint32_t)k << 23)) : 0.f;       // exponent field back to 127: m in [1, 2)
    e = live ? emax + ye + k : ME_EMIN;
    if (valid) buf[(size_t)t * AS] = live ? ptx::lg2(m) + (float)e : NEG_INF;
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Fast path: S <= 32.  Shared-memory rows use a stride of 68 floats (272 B: 16-B aligned for the bulk copies and
// conflict-free when every thread of a quarter-warp reads a float4 of its own row); alpha/beta/emission tables use odd
// strides so that both "lane = state" (phase 1) and "thread = frame" (phase 2) accesses are conflict-free.
constexpr int FAST_THREADS = 64;
constexpr int FAST_XS = 68;

__host__ __device__ inline int fast_alpha_stride(int max_label_len) { return (2 * max_label_len + 1) | 1; }
__host__ __device__ inline int fast_label_stride(int max_label_len) { return max_label_len | 1; }

__global__ void __launch_bounds__(FAST_THREADS, 8)
ctc_fast_kernel(const float* __restrict__ logits, float* __restrict__ grad, const int* __restrict__ flat_labels,
                const int* __restrict__ label_len, const int* __restrict__ input_len, int T, int N, int blank,
                int max_label_len, float grad_scale, float* __restrict__ costs, int recur) {
  extern __shared__ __align__(16) float sm[];
  const int AS = fast_alpha_stride(max_label_len), ES = fast_label_stride(max_label_len);
  float* s_x = sm;                                 // [T][68]  logits -> p -> gradient row
  float* s_alpha = s_x + (size_t)T * FAST_XS;      // [T][AS]
  float* s_beta = s_alpha + (size_t)T * AS;        // [T][AS]
  float* s_el = s_beta + (size_t)T * AS;           // [T][ES]  log2 y_t(label k)
  float* s_eb = s_el + (size_t)T * ES;             // [T]      log2 y_t(blank)
  float* s_k = s_eb + T;                           // [T]      grad_scale / sum_c 2^(x-m)
  __shared__ uint64_t s_bar;
  __shared__ int s_ext[32];
  __shared__ int s_off, s_repeats, s_bad;

  const int n = blockIdx.x, tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int L = label_len[n];
  const int Tn = max(0, min(input_len[n], T));
  const int S = 2 * L + 1;

  if (tid == 0) {
    ptx::mbar_init(&s_bar, FAST_THREADS);
    ptx::fence_barrier_init();
    s_repeats = 0;
    s_bad = 0;
  }
  __syncthreads();
  {   // every thread fetches its own frames; rows past input_len are never read
    const int rows = (Tn > tid) ? (Tn - tid + FAST_THREADS - 1) / FAST_THREADS : 0;
    ptx::mbar_arrive_expect_tx(&s_bar, (uint32_t)rows * CTC_C * (uint32_t)sizeof(float));
    for (int t = tid; t < Tn; t += FAST_THREADS)
      ptx::bulk_load_1d(s_x + (size_t)t * FAST_XS, logits + ((size_t)t * N + n) * CTC_C, CTC_C * sizeof(float), &s_bar);
  }
  // label bookkeeping while the rows are in flight: offset = sum(label_len[0..n)), extended labels, repeat count
  if (warp == 0) {
    int acc = 0;
    for (int i = lane; i < n; i += 32) acc += __ldg(label_len + i);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) s_off = acc;
  }
  __syncthreads();
  bool too_long = (L < 0) || (L > max_label_len) || (S > 32);
  if (!too_long && tid < 32) {
    int v = blank, rep = 0, bad = 0;
    if (tid < S && (tid & 1)) {
      v = flat_labels[s_off + (tid >> 1)];
      // ids outside [0,C) or equal to the blank are never used as row indices: the sample is rejected (cost NaN, zero gradient)
      if (v < 0 || v >= CTC_C || v == blank) { bad = 1; v = blank; }
      if (tid >= 3 && v == flat_labels[s_off + (tid >> 1) - 1]) rep = 1;
    }
    s_ext[tid] = v;
    rep = __popc(__ballot_sync(0xffffffffu, rep));
    bad = __any_sync(0xffffffffu, bad);
    if (tid == 0) { s_repeats = rep; s_bad = bad; }
  }
  __syncthreads();
  too_long = too_long || (s_bad != 0);
  ptx::mbar_wait(&s_bar, 0);                        // also required before an early exit: the copies target this CTA's smem

  const bool feasible = !too_long && Tn > 0 && (L + s_repeats <= Tn);
  if (!feasible) {
    if (tid == 0) costs[n] = too_long ? __int_as_float(0x7fc00000) : 0.0f;
    if (grad != nullptr)
      for (int i = tid; i < T * (CTC_C / 4); i += FAST_THREADS)
        reinterpret_cast<float4*>(grad + ((size_t)(i / (CTC_C / 4)) * N + n) * CTC_C)[i % (CTC_C / 4)] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }

  // ---------------- phase 0: thread = frame ----------------
  for (int t = tid; t < Tn; t += FAST_THREADS) {
    float4* row4 = reinterpret_cast<float4*>(s_x + (size_t)t * FAST_XS);
    const float* row = s_x + (size_t)t * FAST_XS;
    float v[CTC_C];
#pragma unroll
    for (int q = 0; q < CTC_C / 4; ++q) {
      const float4 x = row4[q];
      v[4 * q] = x.x; v[4 * q + 1] = x.y; v[4 * q + 2] = x.z; v[4 * q + 3] = x.w;
    }
    float mx[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) mx[q] = fmaxf(fmaxf(v[4 * q], v[4 * q + 1]), fmaxf(v[4 * q + 2], v[4 * q + 3]));
#pragma unroll
    for (int q = 0; q < 4; ++q) mx[q] = fmaxf(fmaxf(mx[4 * q], mx[4 * q + 1]), fmaxf(mx[4 * q + 2], mx[4 * q + 3]));
    const float mm = fmaxf(fmaxf(mx[0], mx[1]), fmaxf(mx[2], mx[3])) * LOG2E;
    float sum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < CTC_C; ++j) {
      v[j] = ptx::ex2(fmaf(v[j], LOG2E, -mm));
      sum[j & 3] += v[j];
    }
    const float tot = (sum[0] + sum[1]) + (sum[2] + sum[3]);
    const float lse2 = mm + ptx::lg2(tot);
    // emission scores come from the raw logits still in shared memory
    s_eb[t] = fmaf(row[blank], LOG2E, -lse2);
    for (int k = 0; k < L; ++k) s_el[(size_t)t * ES + k] = fmaf(row[s_ext[2 * k + 1]], LOG2E, -lse2);
    s_k[t] = __fdividef(grad_scale, tot);
#pragma unroll
    for (int q = 0; q < CTC_C / 4; ++q) row4[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  }
  __syncthreads();

  // ---------------- phase 1: alpha and reversed beta, one instruction stream ----------------
  if (recur) {
    ctc_recursion_me(s_alpha, s_beta, s_el, s_eb, s_ext, AS, ES, S, Tn, blank, warp, lane);
  } else {
    const bool packed = (S <= 16);
    if (warp < (packed ? 1 : 2)) {
      const int W = packed ? 16 : 32;
      const int half = packed ? (lane >> 4) : warp;            // 0 = alpha, 1 = beta (state order reversed)
      const int j = packed ? (lane & 15) : lane;
      const bool valid = j < S;
      const int s = valid ? (half ? S - 1 - j : j) : 0;
      bool ok2;
      if (half == 0) ok2 = valid && (s >= 2) && (s_ext[s] != blank) && (s_ext[s] != s_ext[s - 2]);
      else           ok2 = valid && (s + 2 < S) && (s_ext[s + 2] != blank) && (s_ext[s + 2] != s_ext[s]);
      const float k1 = (valid && j >= 1) ? 0.f : NEG_INF;
      const float k2 = ok2 ? 0.f : NEG_INF;
      // The transition masks are added by the SENDING lane (k?n = the receiver's mask), so that the three sums leaving the
      // log come out of one FADD level: per step the dependency chain is SHFL, FMNMX3, FADD, EX2, FADD, FADD, LG2, FADD.
      // The shuffles rotate within the W-lane segment; the wrapped-around values carry the masks of lanes 0/1 (= -inf).
      const int seg = lane & ~(W - 1);
      const int src1 = seg | ((j - 1) & (W - 1)), src2 = seg | ((j - 2) & (W - 1));
      const float k1n = __shfl_sync(0xffffffffu, k1, seg | ((j + 1) & (W - 1)));
      const float k2n = __shfl_sync(0xffffffffu, k2, seg | ((j + 2) & (W - 1)));
      float* buf = (half ? s_beta : s_alpha) + s;
      const float* ep = (s & 1) ? (s_el + (s >> 1)) : s_eb;
      const int estride = (s & 1) ? ES : 1;
      const int dt = half ? -1 : 1;
      int t = half ? Tn - 1 : 0;
      float a = (valid && j < 2) ? ep[(size_t)t * estride] : NEG_INF;
      float a1 = a + k1n, a2 = a + k2n;
      if (valid) buf[(size_t)t * AS] = a;
      float e_next = (Tn > 1) ? ep[(size_t)(t + dt) * estride] : 0.f;
      for (int step = 1; step < Tn; ++step) {
        t += dt;
        const float e = e_next;
        if (step + 1 < Tn) e_next = ep[(size_t)(t + dt) * estride];
        const float c = fmaxf(a, -1e30f);                                // clamp keeps (-inf) - (-inf) out of the exponent
        const float u1 = __shfl_sync(0xffffffffu, a1, src1);
        const float u2 = __shfl_sync(0xffffffffu, a2, src2);
        const float m = max3(c, u1, u2);                                 // one FMNMX3 behind the shuffles (c is ready earlier)
        const float sum = ptx::ex2(a - m) + (ptx::ex2(u1 - m) + ptx::ex2(u2 - m));
        const float lg = ptx::lg2(sum), me = m + e;
        a = lg + me;
        a1 = lg + (me + k1n);
        a2 = lg + (me + k2n);
        if (valid) buf[(size_t)t * AS] = a;
      }
    }
  }
  __syncthreads();

  const float aS1 = s_alpha[(size_t)(Tn - 1) * AS + (S - 1)];
  const float aS2 = (S >= 2) ? s_alpha[(size_t)(Tn - 1) * AS + (S - 2)] : NEG_INF;
  const float ll2 = lse3(aS1, aS2, NEG_INF);
  if (tid == 0) costs[n] = -ll2 * LN2;
  if (grad == nullptr) return;

  // ---------------- phase 2: thread = frame, gradient row built in place and bulk-stored ----------------
  for (int t = tid; t < T; t += FAST_THREADS) {
    float4* row4 = reinterpret_cast<float4*>(s_x + (size_t)t * FAST_XS);
    float* row = s_x + (size_t)t * FAST_XS;
    if (t >= Tn || ll2 == NEG_INF) {
#pragma unroll
      for (int q = 0; q < CTC_C / 4; ++q) row4[q] = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      const float k = s_k[t];
#pragma unroll
      for (int q = 0; q < CTC_C / 4; ++q) {
        float4 x = row4[q];
        x.x *= k; x.y *= k; x.z *= k; x.w *= k;
        row4[q] = x;
      }
      const float* al = s_alpha + (size_t)t * AS;
      const float* be = s_beta + (size_t)t * AS;
      const float eb = s_eb[t] + ll2;
      float wb = ptx::ex2(al[0] + be[0] - eb);                       // blank states: one accumulated update
      for (int kk = 0; kk < L; ++kk) {
        const float el = s_el[(size_t)t * ES + kk] + ll2;
        const float w = ptx::ex2(al[2 * kk + 1] + be[2 * kk + 1] - el);   // alpha*beta / y / p(l|x)
        wb += ptx::ex2(al[2 * kk + 2] + be[2 * kk + 2] - eb);
        const int c = s_ext[2 * kk + 1];
        row[c] = fmaf(-grad_scale, w, row[c]);
      }
      row[blank] = fmaf(-grad_scale, wb, row[blank]);
    }
    ptx::fence_proxy_async_smem();
    ptx::bulk_store_1d(grad + ((size_t)t * N + n) * CTC_C, row, CTC_C * sizeof(float));
  }
  ptx::bulk_commit();
  ptx::bulk_wait_read_all();
}


// ---------------------------------------------------------------------------------------------------------------------------
// ctc_tma_kernel: same arithmetic as ctc_fast_kernel, different data movement.  In ctc_fast_kernel every
// thread issues its own `cp.async.bulk` row copies: UBLKCP takes its operands from
// UNIFORM registers, so a warp whose 32 lanes each issue their own row copy executes them one lane at a time (ELECT / R2UR /
// BRA.U.ANY).  Here ONE thread issues two tensor-map loads for the whole utterance -- logits [T,N,64] f32 viewed as
// {32, 2, N, T} with a {32, 1, 1, T} box, i.e. the left and the right 128-byte half of all T rows -- into two 128B-swizzled
// tiles (thread = frame then reads its own 128-byte rows without bank conflicts: chunk q of row t lives at q ^ (t & 7)), and
// the gradient tile leaves through two tensor-map stores.
// ---------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(FAST_THREADS, 8)
ctc_tma_kernel(const __grid_constant__ CUtensorMap tm_logits, const __grid_constant__ CUtensorMap tm_grad, float* __restrict__ grad,
               const int* __restrict__ flat_labels, const int* __restrict__ label_len, const int* __restrict__ input_len, int T, int N,
               int blank, int max_label_len, float grad_scale, float* __restrict__ costs, int tile_rows, int recur) {
  extern __shared__ uint8_t sm_raw[];
  // tile_rows = T rounded up to 8: a half tile is tile_rows x 128 B, both halves 1024-byte aligned
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(sm_raw) + 1023) & ~uintptr_t(1023));
  const int half_floats = tile_rows * 32;
  float* s_x = reinterpret_cast<float*>(base);                 // [2][tile_rows][32] swizzled: logits -> p -> gradient rows
  const int AS = fast_alpha_stride(max_label_len), ES = fast_label_stride(max_label_len);
  float* s_alpha = s_x + 2 * half_floats;          // [T][AS]
  float* s_beta = s_alpha + (size_t)T * AS;        // [T][AS]
  float* s_el = s_beta + (size_t)T * AS;           // [T][ES]  log2 y_t(label k)
  float* s_eb = s_el + (size_t)T * ES;             // [T]      log2 y_t(blank)
  float* s_k = s_eb + T;                           // [T]      grad_scale / sum_c 2^(x-m)
  __shared__ uint64_t s_bar;
  __shared__ int s_ext[32];
  __shared__ int s_off, s_repeats, s_bad;
  auto F4 = [&](int t, int g) { return (g >> 3) * half_floats + t * 32 + (((g & 7) ^ (t & 7)) << 2); };
  auto EL = [&](int t, int c) { return F4(t, c >> 2) + (c & 3); };

  const int n = blockIdx.x, tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int L = label_len[n];
  const int Tn = max(0, min(input_len[n], T));
  const int S = 2 * L + 1;

  if (tid == 0) {
    ptx::prefetch_tmap(&tm_logits);
    ptx::mbar_init(&s_bar, 1);
    ptx::fence_barrier_init();
    s_repeats = 0;
    s_bad = 0;
  }
  __syncthreads();
  if (tid == 0) {
    ptx::mbar_arrive_expect_tx(&s_bar, (uint32_t)(2 * T * 128));
    ptx::tma_load_4d(&tm_logits, &s_bar, s_x, 0, 0, n, 0);
    ptx::tma_load_4d(&tm_logits, &s_bar, s_x + half_floats, 0, 1, n, 0);
  }
  // label bookkeeping while the tile is in flight: offset = sum(label_len[0..n)), extended labels, repeat count
  if (warp == 0) {
    int acc = 0;
    for (int i = lane; i < n; i += 32) acc += __ldg(label_len + i);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) s_off = acc;
  }
  __syncthreads();
  bool too_long = (L < 0) || (L > max_label_len) || (S > 32);
  if (!too_long && tid < 32) {
    int v = blank, rep = 0, bad = 0;
    if (tid < S && (tid & 1)) {
      v = flat_labels[s_off + (tid >> 1)];
      if (v < 0 || v >= CTC_C || v == blank) { bad = 1; v = blank; }
      if (tid >= 3 && v == flat_labels[s_off + (tid >> 1) - 1]) rep = 1;
    }
    s_ext[tid] = v;
    rep = __popc(__ballot_sync(0xffffffffu, rep));
    bad = __any_sync(0xffffffffu, bad);
    if (tid == 0) { s_repeats = rep; s_bad = bad; }
  }
  __syncthreads();
  too_long = too_long || (s_bad != 0);
  ptx::mbar_wait(&s_bar, 0);                        // also required before an early exit: the copies target this CTA's smem

  const bool feasible = !too_long && Tn > 0 && (L + s_repeats <= Tn);
  if (!feasible) {
    if (tid == 0) costs[n] = too_long ? __int_as_float(0x7fc00000) : 0.0f;
    if (grad != nullptr)
      for (int i = tid; i < T * (CTC_C / 4); i += FAST_THREADS)
        reinterpret_cast<float4*>(grad + ((size_t)(i / (CTC_C / 4)) * N + n) * CTC_C)[i % (CTC_C / 4)] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }

  // ---------------- phase 0: thread = frame ----------------
  for (int t = tid; t < Tn; t += FAST_THREADS) {
    float v[CTC_C];
#pragma unroll
    for (int g = 0; g < CTC_C / 4; ++g) {
      const float4 x = *reinterpret_cast<const float4*>(s_x + F4(t, g));
      v[4 * g] = x.x; v[4 * g + 1] = x.y; v[4 * g + 2] = x.z; v[4 * g + 3] = x.w;
    }
    float mx[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) mx[q] = fmaxf(fmaxf(v[4 * q], v[4 * q + 1]), fmaxf(v[4 * q + 2], v[4 * q + 3]));
#pragma unroll
    for (int q = 0; q < 4; ++q) mx[q] = fmaxf(fmaxf(mx[4 * q], mx[4 * q + 1]), fmaxf(mx[4 * q + 2], mx[4 * q + 3]));
    const float mm = fmaxf(fmaxf(mx[0], mx[1]), fmaxf(mx[2], mx[3])) * LOG2E;
    float sum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < CTC_C; ++j) {
      v[j] = ptx::ex2(fmaf(v[j], LOG2E, -mm));
      sum[j & 3] += v[j];
    }
    const float tot = (sum[0] + sum[1]) + (sum[2] + sum[3]);
    const float lse2 = mm + ptx::lg2(tot);
    // emission scores come from the raw logits still in shared memory
    s_eb[t] = fmaf(s_x[EL(t, blank)], LOG2E, -lse2);
    for (int k = 0; k < L; ++k) s_el[(size_t)t * ES + k] = fmaf(s_x[EL(t, s_ext[2 * k + 1])], LOG2E, -lse2);
    s_k[t] = __fdividef(grad_scale, tot);
#pragma unroll
    for (int g = 0; g < CTC_C / 4; ++g)
      *reinterpret_cast<float4*>(s_x + F4(t, g)) = make_float4(v[4 * g], v[4 * g + 1], v[4 * g + 2], v[4 * g + 3]);
  }
  __syncthreads();

  // ---------------- phase 1: alpha and reversed beta, one instruction stream (identical to ctc_fast_kernel) ----------------
  if (recur) {
    ctc_recursion_me(s_alpha, s_beta, s_el, s_eb, s_ext, AS, ES, S, Tn, blank, warp, lane);
  } else {
    const bool packed = (S <= 16);
    if (warp < (packed ? 1 : 2)) {
      const int W = packed ? 16 : 32;
      const int half = packed ? (lane >> 4) : warp;            // 0 = alpha, 1 = beta (state order reversed)
      const int j = packed ? (lane & 15) : lane;
      const bool valid = j < S;
      const int s = valid ? (half ? S - 1 - j : j) : 0;
      bool ok2;
      if (half == 0) ok2 = valid && (s >= 2) && (s_ext[s] != blank) && (s_ext[s] != s_ext[s - 2]);
      else           ok2 = valid && (s + 2 < S) && (s_ext[s + 2] != blank) && (s_ext[s + 2] != s_ext[s]);
      const float k1 = (valid && j >= 1) ? 0.f : NEG_INF;
      const float k2 = ok2 ? 0.f : NEG_INF;
      const int seg = lane & ~(W - 1);
      const int src1 = seg | ((j - 1) & (W - 1)), src2 = seg | ((j - 2) & (W - 1));
      const float k1n = __shfl_sync(0xffffffffu, k1, seg | ((j + 1) & (W - 1)));
      const float k2n = __shfl_sync(0xffffffffu, k2, seg | ((j + 2) & (W - 1)));
      float* buf = (half ? s_beta : s_alpha) + s;
      const float* ep = (s & 1) ? (s_el + (s >> 1)) : s_eb;
      const int estride = (s & 1) ? ES : 1;
      const int dt = half ? -1 : 1;
      int t = half ? Tn - 1 : 0;
      float a = (valid && j < 2) ? ep[(size_t)t * estride] : NEG_INF;
      float a1 = a + k1n, a2 = a + k2n;
      if (valid) buf[(size_t)t * AS] = a;
      float e_next = (Tn > 1) ? ep[(size_t)(t + dt) * estride] : 0.f;
      for (int step = 1; step < Tn; ++step) {
        t += dt;
        const float e = e_next;
        if (step + 1 < Tn) e_next = ep[(size_t)(t + dt) * estride];
        const float c = fmaxf(a, -1e30f);
        const float u1 = __shfl_sync(0xffffffffu, a1, src1);
        const float u2 = __shfl_sync(0xffffffffu, a2, src2);
        const float m = max3(c, u1, u2);
        const float sum = ptx::ex2(a - m) + (ptx::ex2(u1 - m) + ptx::ex2(u2 - m));
        const float lg = ptx::lg2(sum), me = m + e;
        a = lg + me;
        a1 = lg + (me + k1n);
        a2 = lg + (me + k2n);
        if (valid) buf[(size_t)t * AS] = a;
      }
    }
  }
  __syncthreads();

  const float aS1 = s_alpha[(size_t)(Tn - 1) * AS + (S - 1)];
  const float aS2 = (S >= 2) ? s_alpha[(size_t)(Tn - 1) * AS + (S - 2)] : NEG_INF;
  const float ll2 = lse3(aS1, aS2, NEG_INF);
  if (tid == 0) costs[n] = -ll2 * LN2;
  if (grad == nullptr) return;

  // ---------------- phase 2: thread = frame, gradient rows built in place, two tensor-map stores for the utterance ----------------
  for (int t = tid; t < T; t += FAST_THREADS) {
    if (t >= Tn || ll2 == NEG_INF) {
#pragma unroll
      for (int g = 0; g < CTC_C / 4; ++g) *reinterpret_cast<float4*>(s_x + F4(t, g)) = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      const float k = s_k[t];
#pragma unroll
      for (int g = 0; g < CTC_C / 4; ++g) {
        float4 x = *reinterpret_cast<float4*>(s_x + F4(t, g));
        x.x *= k; x.y *= k; x.z *= k; x.w *= k;
        *reinterpret_cast<float4*>(s_x + F4(t, g)) = x;
      }
      const float* al = s_alpha + (size_t)t * AS;
      const float* be = s_beta + (size_t)t * AS;
      const float eb = s_eb[t] + ll2;
      float wb = ptx::ex2(al[0] + be[0] - eb);                       // blank states: one accumulated update
      for (int kk = 0; kk < L; ++kk) {
        const float el = s_el[(size_t)t * ES + kk] + ll2;
        const float w = ptx::ex2(al[2 * kk + 1] + be[2 * kk + 1] - el);   // alpha*beta / y / p(l|x)
        wb += ptx::ex2(al[2 * kk + 2] + be[2 * kk + 2] - eb);
        const int ci = EL(t, s_ext[2 * kk + 1]);
        s_x[ci] = fmaf(-grad_scale, w, s_x[ci]);
      }
      const int bi = EL(t, blank);
      s_x[bi] = fmaf(-grad_scale, wb, s_x[bi]);
    }
  }
  ptx::fence_proxy_async_smem();                    // generic-proxy writes of the tile -> visible to the TMA store
  __syncthreads();
  if (tid == 0) {
    ptx::tma_store_4d(&tm_grad, s_x, 0, 0, n, 0);
    ptx::tma_store_4d(&tm_grad, s_x + half_floats, 0, 1, n, 0);
    ptx::bulk_commit();
    ptx::bulk_wait_read_all();
  }
}

size_t ctc_tma_smem_bytes(int T, int max_label_len) {
  const int tile_rows = (T + 7) / 8 * 8;
  return 1024 + (size_t)2 * tile_rows * 128 +
         sizeof(float) * (size_t)T * (2 * fast_alpha_stride(max_label_len) + fast_label_stride(max_label_len) + 2);
}

size_t ctc_fast_smem_bytes(int T, int max_label_len) {
  return sizeof(float) * (size_t)T * (FAST_XS + 2 * fast_alpha_stride(max_label_len) + fast_label_stride(max_label_len) + 2);
}

// Greedy decode: one warp per utterance, lane = frame (chunks of 32 frames).  VEC: logits 16-byte aligned (float4 row
// loads); otherwise the same values are read one float at a time.
template <bool VEC>
__global__ void __launch_bounds__(128) ctc_greedy_kernel(const float* __restrict__ logits,
                                                         const int* __restrict__ input_len, int T, int N,
                                                         int tf_blank, int strip, int* __restrict__ out,
                                                         int* __restrict__ out_len) {
  const int n = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  int Tn = max(0, min(input_len[n], T));
  int count = 0;
  int prev_carry = -1;
  for (int t0 = 0; t0 < Tn; t0 += 32) {
    int t = t0 + lane;
    int best = -1;
    if (t < Tn) {
      const float* row = logits + ((size_t)t * N + n) * CTC_C;
      float bv = -INFINITY;
      best = 0;
#pragma unroll
      for (int q = 0; q < CTC_C / 4; ++q) {
        const float4 v = VEC ? __ldg(reinterpret_cast<const float4*>(row) + q)
                             : make_float4(__ldg(row + 4 * q), __ldg(row + 4 * q + 1), __ldg(row + 4 * q + 2), __ldg(row + 4 * q + 3));
        if (v.x > bv) { bv = v.x; best = 4 * q; }
        if (v.y > bv) { bv = v.y; best = 4 * q + 1; }
        if (v.z > bv) { bv = v.z; best = 4 * q + 2; }
        if (v.w > bv) { bv = v.w; best = 4 * q + 3; }
      }
      // NaN rows: comparisons false -> best stays 0 (lowest index), matching argmax-on-ties
    }
    int prev = __shfl_up_sync(0xffffffffu, best, 1);
    if (lane == 0) prev = prev_carry;
    bool keep = (t < Tn) && (best != tf_blank) && (best != prev) && (best != strip);
    unsigned m = __ballot_sync(0xffffffffu, keep);
    if (keep) out[(size_t)n * T + count + __popc(m & ((1u << lane) - 1))] = best;
    count += __popc(m);
    prev_carry = __shfl_sync(0xffffffffu, best, 31);
  }
  for (int i = count + lane; i < T; i += 32) out[(size_t)n * T + i] = 0;
  if (lane == 0) out_len[n] = count;
}

// ---------------------------------------------------------------------------------------------------------------------------
// ctc_long_kernel: the workspace path, for max_label_len <= 639 (S <= 1279 states) and any T the workspace holds -- the
// shapes whose alpha / beta tables do not fit in shared memory.  Same semantics and log2-space arithmetic as the kernels
// above.  One CTA of 320 threads per utterance, 4 consecutive states per thread (S_pad <= 1280).
//   prologue  warp = frame: log2-softmax of each frame's 64 logits -> workspace row lp[t][64]
//   alpha     one frame per step: the previous row ping-pongs in shared memory (one barrier per frame); each row is also
//             stored to the workspace.  The next frames' emissions are loaded two steps ahead, off the dependency chain.
//   beta      recomputed row by row from T-1 down; at each frame every state's posterior alpha*beta/y/p against the stored
//             alpha row goes to a shared row, and the frame's gradient row is formed one step later: each class sums its
//             posteriors over a per-utterance class -> state list (built once, in label order), the blank over its L+1 even
//             states, a lane-strided sum then a fixed xor tree.  No float atomics: the result is the same bits run to run.
// Logits and gradient are read and written one float at a time (4-byte alignment is enough).
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int LONG_MAX_LABEL = 639;
constexpr int LONG_MAX_THREADS = 320;
constexpr int LONG_WS_ALIGN = 256;           // the launch rounds the workspace pointer up to this; the size query includes it

inline int long_stride(int max_label_len) { return (2 * max_label_len + 1 + 3) & ~3; }            // S_pad, a multiple of 4
inline size_t long_smem_bytes(int max_label_len) {
  const size_t AS = long_stride(max_label_len);
  return sizeof(float) * (2 * (AS + 8) + 2 * AS) + sizeof(int) * (AS + (size_t)(max_label_len > 0 ? max_label_len : 1) + 65);
}

__global__ void __launch_bounds__(LONG_MAX_THREADS)
ctc_long_kernel(const float* __restrict__ logits, float* __restrict__ grad, const int* __restrict__ flat_labels,
                const int* __restrict__ label_len, const int* __restrict__ input_len, int T, int N, int blank, int max_label_len,
                float grad_scale, float* __restrict__ costs, float* __restrict__ ws) {
  extern __shared__ __align__(16) float lsm[];
  const int AS = (2 * max_label_len + 1 + 3) & ~3;
  const int BS = AS + 8;                              // a row: 4 pad, AS states, 4 pad (pads stay -inf)
  float* s_buf = lsm;                                 // [2][BS] alpha, then beta rows
  float* s_w = s_buf + 2 * BS;                        // [2][AS] posteriors of one frame
  int* s_ext = reinterpret_cast<int*>(s_w + 2 * AS);  // [AS] class of each state (blank past S)
  int* s_list = s_ext + AS;                           // [max_label_len] odd states grouped by class, in label order
  int* s_cstart = s_list + (max_label_len > 0 ? max_label_len : 1);   // [65] class c's states: s_list[s_cstart[c] .. s_cstart[c+1])
  __shared__ int s_off, s_repeats, s_bad;

  const int n = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int warp = tid >> 5, lane = tid & 31, nw = nt >> 5;
  const int L = label_len[n];
  const int Tn = max(0, min(input_len[n], T));
  const int S = 2 * L + 1;
  float* lp = ws + (size_t)n * T * CTC_C;                               // [T][64] log2 y
  float* al = ws + (size_t)N * T * CTC_C + (size_t)n * T * AS;          // [T][AS] log2 alpha

  if (warp == 0) {
    int acc = 0;
    for (int i = lane; i < n; i += 32) acc += __ldg(label_len + i);
    acc = __reduce_add_sync(0xffffffffu, acc);
    if (lane == 0) { s_off = acc; s_repeats = 0; s_bad = 0; }
  }
  __syncthreads();
  bool too_long = (L < 0) || (L > max_label_len);
  if (!too_long) {
    int rep = 0, bad = 0;
    for (int s = tid; s < AS; s += nt) {
      int v = blank;
      if (s < S && (s & 1)) {
        v = flat_labels[s_off + (s >> 1)];
        // ids outside [0,C) or equal to the blank are never used as indices: the sample is rejected (cost NaN, zero gradient)
        if (v < 0 || v >= CTC_C || v == blank) { bad = 1; v = blank; }
        if (s >= 3 && v == flat_labels[s_off + (s >> 1) - 1]) rep++;
      }
      s_ext[s] = v;
    }
    if (rep) atomicAdd(&s_repeats, rep);
    if (bad) atomicOr(&s_bad, 1);
  }
  __syncthreads();
  too_long = too_long || (s_bad != 0);
  const bool feasible = !too_long && Tn > 0 && (L + s_repeats <= Tn);
  if (!feasible) {
    if (tid == 0) costs[n] = too_long ? __int_as_float(0x7fc00000) : 0.0f;
    if (grad != nullptr)
      for (int i = tid; i < T * CTC_C; i += nt) grad[((size_t)(i / CTC_C) * N + n) * CTC_C + (i % CTC_C)] = 0.f;
    return;
  }

  if (grad != nullptr) {   // class -> state lists: count, exclusive scan, fill (ballot order = label order)
    for (int c = warp; c < CTC_C; c += nw) {
      int cnt = 0;
      for (int k0 = 0; k0 < L; k0 += 32) cnt += __popc(__ballot_sync(0xffffffffu, k0 + lane < L && s_ext[2 * (k0 + lane) + 1] == c));
      if (lane == 0) s_cstart[c] = cnt;
    }
    __syncthreads();
    if (tid == 0) {
      int acc = 0;
      for (int c = 0; c < CTC_C; ++c) { const int v = s_cstart[c]; s_cstart[c] = acc; acc += v; }
      s_cstart[CTC_C] = acc;
    }
    __syncthreads();
    for (int c = warp; c < CTC_C; c += nw) {
      int pos = s_cstart[c];
      for (int k0 = 0; k0 < L; k0 += 32) {
        const int k = k0 + lane;
        const bool hit = k < L && s_ext[2 * k + 1] == c;
        const unsigned b = __ballot_sync(0xffffffffu, hit);
        if (hit) s_list[pos + __popc(b & ((1u << lane) - 1))] = 2 * k + 1;
        pos += __popc(b);
      }
    }
  }

  // ---------------- prologue: warp = frame, log2-softmax rows to the workspace ----------------
  for (int t0 = warp; t0 < Tn; t0 += 4 * nw) {
    float x0[4], x1[4], m[4], sum[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int t = min(t0 + u * nw, Tn - 1);
      const float* x = logits + ((size_t)t * N + n) * CTC_C;
      x0[u] = __ldg(x + lane) * LOG2E;
      x1[u] = __ldg(x + lane + 32) * LOG2E;
      m[u] = fmaxf(x0[u], x1[u]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
      for (int u = 0; u < 4; ++u) m[u] = fmaxf(m[u], __shfl_xor_sync(0xffffffffu, m[u], o));
#pragma unroll
    for (int u = 0; u < 4; ++u) sum[u] = ptx::ex2(x0[u] - m[u]) + ptx::ex2(x1[u] - m[u]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
      for (int u = 0; u < 4; ++u) sum[u] += __shfl_xor_sync(0xffffffffu, sum[u], o);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int t = t0 + u * nw;
      const float lse = m[u] + ptx::lg2(sum[u]);
      if (t < Tn) {
        lp[(size_t)t * CTC_C + lane] = x0[u] - lse;
        lp[(size_t)t * CTC_C + lane + 32] = x1[u] - lse;
      }
    }
  }
  for (int i = tid; i < 2 * BS; i += nt) s_buf[i] = NEG_INF;
  __syncthreads();

  const int s0 = 4 * tid;                    // this thread's states s0 .. s0+3 (none when s0 >= AS)
  const bool act = s0 < AS;
  int cls[4];
  bool skin[4], skout[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int s = s0 + k;
    cls[k] = act ? s_ext[s] : blank;
    skin[k] = act && s >= 2 && s < S && s_ext[s] != blank && s_ext[s] != s_ext[s - 2];
    skout[k] = act && s + 2 < S && s_ext[s + 2] != blank && s_ext[s + 2] != s_ext[s];
  }
  auto emit = [&](int t, float* e) {
#pragma unroll
    for (int k = 0; k < 4; ++k) e[k] = lp[(size_t)t * CTC_C + cls[k]];
  };

  // ---------------- alpha ----------------
  float a[4], e1[4] = {0.f, 0.f, 0.f, 0.f}, e2[4] = {0.f, 0.f, 0.f, 0.f};
  if (act) {
    float e0[4];
    emit(0, e0);
#pragma unroll
    for (int k = 0; k < 4; ++k) a[k] = (s0 + k < 2 && s0 + k < S) ? e0[k] : NEG_INF;
    const float4 v = make_float4(a[0], a[1], a[2], a[3]);
    *reinterpret_cast<float4*>(s_buf + 4 + s0) = v;
    *reinterpret_cast<float4*>(al + s0) = v;
    if (Tn > 1) emit(1, e1);
    if (Tn > 2) emit(2, e2);
  }
  __syncthreads();
  for (int t = 1; t < Tn; ++t) {
    if (act) {
      const float* prev = s_buf + ((t - 1) & 1) * BS;
      float* cur = s_buf + (t & 1) * BS;
      float e[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) { e[k] = e1[k]; e1[k] = e2[k]; }
      if (t + 2 < Tn) emit(t + 2, e2);
      const float2 lo = *reinterpret_cast<const float2*>(prev + 4 + s0 - 2);     // states s0-2, s0-1
      const float v[6] = {lo.x, lo.y, a[0], a[1], a[2], a[3]};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float nv = lse3(v[k + 2], v[k + 1], skin[k] ? v[k] : NEG_INF) + e[k];
        a[k] = (s0 + k < S) ? nv : NEG_INF;
      }
      const float4 o = make_float4(a[0], a[1], a[2], a[3]);
      *reinterpret_cast<float4*>(cur + 4 + s0) = o;
      *reinterpret_cast<float4*>(al + (size_t)t * AS + s0) = o;
    }
    __syncthreads();
  }

  const float* last = s_buf + ((Tn - 1) & 1) * BS + 4;
  const float ll2 = lse3(last[S - 1], (S >= 2) ? last[S - 2] : NEG_INF, NEG_INF);
  if (tid == 0) costs[n] = -ll2 * LN2;
  if (grad == nullptr) return;
  {
    const int z0 = (ll2 == NEG_INF) ? 0 : Tn;      // frames past the length (all of them when p underflows) get zero
    for (int i = tid; i < (T - z0) * CTC_C; i += nt) grad[((size_t)(z0 + i / CTC_C) * N + n) * CTC_C + (i % CTC_C)] = 0.f;
  }
  if (ll2 == NEG_INF) return;
  __syncthreads();                                  // every thread has read the last alpha row

  // ---------------- beta, posteriors, gradient rows ----------------
  // The gradient row of frame t+1 is formed while beta of frame t is computed: lane j of warp w owns class w + nw*j.
  const int ncls = (CTC_C + nw - 1) / nw;
  auto ycls = [&](int t) { const int c = warp + nw * lane; return (lane < ncls && c < CTC_C) ? lp[(size_t)t * CTC_C + c] : 0.f; };
  auto grad_row = [&](int t, const float* sw, float yl) {
    float* g = grad + ((size_t)t * N + n) * CTC_C;
    for (int j = 0; j < ncls; ++j) {
      const int c = warp + nw * j;
      if (c >= CTC_C) break;
      float acc = 0.f;
      if (c == blank) {
        for (int i = lane; i <= L; i += 32) acc += sw[2 * i];
      } else {
        for (int i = s_cstart[c] + lane; i < s_cstart[c + 1]; i += 32) acc += sw[s_list[i]];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == j) g[c] = grad_scale * (ptx::ex2(yl) - acc);
    }
  };
  float b[4], ec[4], en1[4] = {0.f, 0.f, 0.f, 0.f}, en2[4] = {0.f, 0.f, 0.f, 0.f};
  float4 ac = make_float4(0.f, 0.f, 0.f, 0.f), an1 = ac, an2 = ac;
  if (act) {
    emit(Tn - 1, ec);
    ac = *reinterpret_cast<const float4*>(al + (size_t)(Tn - 1) * AS + s0);
    if (Tn > 1) { emit(Tn - 2, en1); an1 = *reinterpret_cast<const float4*>(al + (size_t)(Tn - 2) * AS + s0); }
    if (Tn > 2) { emit(Tn - 3, en2); an2 = *reinterpret_cast<const float4*>(al + (size_t)(Tn - 3) * AS + s0); }
  }
  float ynext = ycls(Tn - 1), ycur = 0.f;
  for (int t = Tn - 1; t >= 0; --t) {
    const float yrow = ycur;                        // class values of frame t+1
    ycur = ynext;
    if (t > 0) ynext = ycls(t - 1);
    if (act) {
      const float* prev = s_buf + ((t + 1) & 1) * BS;
      float* cur = s_buf + (t & 1) * BS;
      if (t == Tn - 1) {
#pragma unroll
        for (int k = 0; k < 4; ++k) b[k] = (s0 + k < S && s0 + k >= S - 2) ? ec[k] : NEG_INF;
      } else {
        const float2 hi = *reinterpret_cast<const float2*>(prev + 4 + s0 + 4);   // states s0+4, s0+5
        const float v[6] = {b[0], b[1], b[2], b[3], hi.x, hi.y};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float nv = lse3(v[k], v[k + 1], skout[k] ? v[k + 2] : NEG_INF) + ec[k];
          b[k] = (s0 + k < S) ? nv : NEG_INF;
        }
      }
      *reinterpret_cast<float4*>(cur + 4 + s0) = make_float4(b[0], b[1], b[2], b[3]);
      const float av[4] = {ac.x, ac.y, ac.z, ac.w};
      float w[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) w[k] = ptx::ex2(av[k] + b[k] - ec[k] - ll2);   // alpha*beta / y / p(l|x)
      *reinterpret_cast<float4*>(s_w + (t & 1) * AS + s0) = make_float4(w[0], w[1], w[2], w[3]);
#pragma unroll
      for (int k = 0; k < 4; ++k) { ec[k] = en1[k]; en1[k] = en2[k]; }
      ac = an1; an1 = an2;
      if (t >= 3) { emit(t - 3, en2); an2 = *reinterpret_cast<const float4*>(al + (size_t)(t - 3) * AS + s0); }
    }
    if (t + 1 < Tn) grad_row(t + 1, s_w + ((t + 1) & 1) * AS, yrow);
    __syncthreads();
  }
  grad_row(0, s_w, ycur);
}

size_t ctc_smem_bytes(int T, int KS) { return sizeof(float) * ((size_t)T + 3 * (size_t)T * 32 * KS + CTC_WARPS * 4 * CTC_C); }

template <int KS>
int launch_ctc(const float* logits, float* grad, const int* flat_labels, const int* label_len, const int* input_len,
               int T, int N, int blank, float grad_scale, float* costs, cudaStream_t st, const char* more) {
  size_t smem = ctc_smem_bytes(T, KS);
  if (smem > 200 * 1024)
    return crnn_fail(CRNN_UNSUPPORTED, "ctc_loss: T = %d frames need %zu bytes of shared memory at KS = %d (limit %d)%s", T, smem, KS,
                     200 * 1024, more);
  CUDA_TRY(cudaFuncSetAttribute(ctc_loss_kernel<KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ctc_loss_kernel<KS><<<N, CTC_THREADS, smem, st>>>(logits, grad, flat_labels, label_len, input_len, T, N, blank, grad_scale,
                                           costs);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}

// CRNN_CTC_KERNEL=generic routes S <= 32 to ctc_loss_kernel<1> as well (the parity tests run both kernels on the same inputs).
bool ctc_force_generic() {
  const char* e = getenv("CRNN_CTC_KERNEL");
  return e != nullptr && strcmp(e, "generic") == 0;
}

// [T, N, 64] f32 viewed as {32, 2, N, T}: box = the left or right 128-byte half of all T rows of one utterance, 128B swizzle
int make_tmap_ctc(CUtensorMap* m, const float* base, int T, int N) {
  typedef CUresult (*PFN)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                          const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static PFN enc = nullptr;
  if (!enc) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled unavailable");
    enc = reinterpret_cast<PFN>(p);
  }
  cuuint64_t dims[4] = {32, 2, (cuuint64_t)N, (cuuint64_t)T};
  cuuint64_t strides[3] = {128, 256, (cuuint64_t)N * 256};
  cuuint32_t box[4] = {32, 1, 1, (cuuint32_t)T};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled(ctc) failed: %d", (int)r);
  return CRNN_OK;
}

// which S <= 32 kernel: "fast" (default: per-thread bulk row copies), "tma" (one tensor-map tile load/store per utterance, kept
// selectable and tested), "generic"
int ctc_kernel_choice() {
  const char* e = getenv("CRNN_CTC_KERNEL");
  if (e != nullptr && strcmp(e, "generic") == 0) return 2;
  if (e != nullptr && strcmp(e, "tma") == 0) return 0;
  return 1;
}
// alpha/beta recursion of the S <= 32 kernels: "log" (default: log2-space, 3 EX2 + 1 LG2 per step) or "me" (mantissa/exponent pairs:
// no transcendental on the chain and ~1e-8 relative accuracy instead of ~1e-5, but MORE dependent integer/select instructions per
// step, so it is the accuracy option, not the speed option)
int ctc_recur_choice() {
  const char* e = getenv("CRNN_CTC_RECUR");
  return (e != nullptr && strcmp(e, "me") == 0) ? 1 : 0;
}

// CRNN_CTC_KERNEL=long runs ctc_long_kernel at every shape (the size query then returns its bytes everywhere), so that the
// workspace kernel can be checked at the shapes the shared-memory kernels serve
bool ctc_force_long() {
  const char* e = getenv("CRNN_CTC_KERNEL");
  return e != nullptr && strcmp(e, "long") == 0;
}

// states-per-lane variant of the generic kernel, and whether its shared memory holds T frames (every alignment)
int ctc_generic_ks(int max_label_len) {
  const int S = 2 * max_label_len + 1;
  return S <= 32 ? 1 : S <= 64 ? 2 : S <= 128 ? 4 : 0;
}
bool ctc_generic_fits(int T, int max_label_len) {
  const int ks = ctc_generic_ks(max_label_len);
  return ks != 0 && ctc_smem_bytes(T, ks) <= 200 * 1024;
}

// Workspace of ctc_long_kernel: per utterance T log2-softmax rows (64 floats) and T alpha rows (S_pad floats), plus the
// alignment slack.  The per-utterance float count must fit an int; the total must fit a size_t.  No crnn_fail here.
int ctc_long_bytes(int T, int N, int max_label_len, size_t* bytes) {
  if (max_label_len > LONG_MAX_LABEL) return CRNN_UNSUPPORTED;
  const size_t per = (size_t)T * (size_t)(CTC_C + long_stride(max_label_len));
  if (per > (size_t)INT_MAX || per > (SIZE_MAX - LONG_WS_ALIGN) / sizeof(float) / (size_t)N) return CRNN_UNSUPPORTED;
  *bytes = per * (size_t)N * sizeof(float) + LONG_WS_ALIGN;
  return CRNN_OK;
}

int launch_ctc_long(const float* logits, float* grad, const int* flat_labels, const int* label_len, const int* input_len, int T,
                    int N, int blank, int max_label_len, float grad_scale, float* costs, void* workspace, cudaStream_t st) {
  float* ws = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(workspace) + LONG_WS_ALIGN - 1) & ~uintptr_t(LONG_WS_ALIGN - 1));
  // always 320 threads: short labels leave threads idle in the recursions, but the per-frame class sums still get 10 warps
  ctc_long_kernel<<<N, LONG_MAX_THREADS, long_smem_bytes(max_label_len), st>>>(
      logits, grad, flat_labels, label_len, input_len, T, N, blank, max_label_len, grad_scale, costs, ws);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}

}  // namespace

extern "C" int crnn_ctc_workspace_size(int T, int N, int C, int max_label_len, size_t* bytes) {
  if (!bytes || T <= 0 || N <= 0 || max_label_len < 0) return crnn_fail(CRNN_INVALID_VALUE, "ctc_workspace_size: bad args");
  if (C != CTC_C) return crnn_fail(CRNN_UNSUPPORTED, "ctc: C must be 64");
  if (ctc_generic_fits(T, max_label_len) && !ctc_force_long()) {
    *bytes = 0;   // a shared-memory kernel serves the shape at any alignment
    return CRNN_OK;
  }
  size_t need = 0;
  if (ctc_long_bytes(T, N, max_label_len, &need) != CRNN_OK)
    return crnn_fail(CRNN_UNSUPPORTED, "ctc_workspace_size: max_label_len = %d, T = %d, N = %d is beyond the workspace kernel "
                     "(max_label_len <= %d, per-utterance and total sizes within int / size_t)", max_label_len, T, N, LONG_MAX_LABEL);
  *bytes = need;
  return CRNN_OK;
}

extern "C" int crnn_ctc_loss(const float* logits, float* grad, const int* flat_labels, const int* label_len,
                             const int* input_len, int T, int N, int C, int blank, int max_label_len,
                             float grad_scale, float* costs, void* workspace, size_t workspace_bytes,
                             crnn_stream_t stream) {
  if (!logits || !flat_labels || !label_len || !input_len || !costs) return crnn_fail(CRNN_INVALID_VALUE, "ctc_loss: null pointer");
  if (T <= 0 || N <= 0 || blank < 0 || blank >= C || max_label_len < 0) return crnn_fail(CRNN_INVALID_VALUE, "ctc_loss: bad shape");
  if (C != CTC_C) return crnn_fail(CRNN_UNSUPPORTED, "ctc: C must be 64");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int S = 2 * max_label_len + 1;
  // The workspace kernel runs only where no shared-memory kernel can (or when forced): every other call takes the kernel
  // and computes the bits it would without a workspace.
  size_t need = 0;
  const bool long_ok = ctc_long_bytes(T, N, max_label_len, &need) == CRNN_OK;
  const bool force_long = ctc_force_long();
  if (force_long) {
    if (long_ok && workspace != nullptr && workspace_bytes >= need)
      return launch_ctc_long(logits, grad, flat_labels, label_len, input_len, T, N, blank, max_label_len, grad_scale, costs, workspace, st);
    if (!long_ok)
      return crnn_fail(CRNN_UNSUPPORTED, "ctc_loss: CRNN_CTC_KERNEL=long: max_label_len = %d, T = %d is beyond the workspace kernel",
                       max_label_len, T);
    return crnn_fail(CRNN_UNSUPPORTED, "ctc_loss: CRNN_CTC_KERNEL=long needs a workspace of %zu bytes, got %zu", need,
                     workspace != nullptr ? workspace_bytes : (size_t)0);
  }
  const bool aligned = (reinterpret_cast<uintptr_t>(logits) % 16 == 0) && (grad == nullptr || reinterpret_cast<uintptr_t>(grad) % 16 == 0);
  if (S <= 32 && aligned && T <= 256 && ctc_kernel_choice() == 0 && ctc_tma_smem_bytes(T, max_label_len) <= 200 * 1024) {
    CUtensorMap tl, tg;
    CRNN_TRY(make_tmap_ctc(&tl, logits, T, N));
    CRNN_TRY(make_tmap_ctc(&tg, grad != nullptr ? grad : logits, T, N));
    const size_t smem = ctc_tma_smem_bytes(T, max_label_len);
    static size_t attr_smem = 0;
    if (smem > attr_smem) {
      CUDA_TRY(cudaFuncSetAttribute(ctc_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      attr_smem = smem;
    }
    ctc_tma_kernel<<<N, FAST_THREADS, smem, st>>>(tl, tg, grad, flat_labels, label_len, input_len, T, N, blank, max_label_len, grad_scale,
                                                  costs, (T + 7) / 8 * 8, ctc_recur_choice());
    CUDA_TRY(cudaGetLastError());
    return CRNN_OK;
  }
  if (S <= 32 && aligned && ctc_fast_smem_bytes(T, max_label_len) <= 200 * 1024 && !ctc_force_generic()) {
    const size_t smem = ctc_fast_smem_bytes(T, max_label_len);
    CUDA_TRY(cudaFuncSetAttribute(ctc_fast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ctc_fast_kernel<<<N, FAST_THREADS, smem, st>>>(logits, grad, flat_labels, label_len, input_len, T, N, blank, max_label_len,
                                                   grad_scale, costs, ctc_recur_choice());
    CUDA_TRY(cudaGetLastError());
    return CRNN_OK;
  }
  const bool run_long = !ctc_generic_fits(T, max_label_len) && long_ok && workspace != nullptr && workspace_bytes >= need;
  if (run_long)
    return launch_ctc_long(logits, grad, flat_labels, label_len, input_len, T, N, blank, max_label_len, grad_scale, costs, workspace, st);
  // no kernel runs: the failure names what the shared-memory kernels needed and, in range, the workspace that would run it
  char more[96] = "";
  if (long_ok) snprintf(more, sizeof more, "; a workspace of %zu bytes runs it", need);
  if (S <= 32) return launch_ctc<1>(logits, grad, flat_labels, label_len, input_len, T, N, blank, grad_scale, costs, st, more);
  if (S <= 64) return launch_ctc<2>(logits, grad, flat_labels, label_len, input_len, T, N, blank, grad_scale, costs, st, more);
  if (S <= 128) return launch_ctc<4>(logits, grad, flat_labels, label_len, input_len, T, N, blank, grad_scale, costs, st, more);
  return crnn_fail(CRNN_UNSUPPORTED, "ctc: max_label_len > 63%s", more);
}

extern "C" int crnn_ctc_greedy(const float* logits, const int* input_len, int T, int N, int C, int tf_blank,
                               int strip, int* out, int* out_len, crnn_stream_t stream) {
  if (!logits || !input_len || !out || !out_len || T <= 0 || N <= 0) return crnn_fail(CRNN_INVALID_VALUE, "ctc_greedy: bad args");
  if (C != CTC_C) return crnn_fail(CRNN_UNSUPPORTED, "ctc: C must be 64");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (reinterpret_cast<uintptr_t>(logits) % 16 == 0)
    ctc_greedy_kernel<true><<<(N + 3) / 4, 128, 0, st>>>(logits, input_len, T, N, tf_blank, strip, out, out_len);
  else
    ctc_greedy_kernel<false><<<(N + 3) / 4, 128, 0, st>>>(logits, input_len, T, N, tf_blank, strip, out, out_len);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
