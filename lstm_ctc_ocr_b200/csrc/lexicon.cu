// Lexicon-based reading (CRNN's lexicon transcription, Shi, Bai & Yao 2015, §2.3.2) for C = 64 classes, sm_90a: the lexicon
// entries nearest a line's read by edit distance, and the CTC probability of each such entry under the line's frames.
//
// lexicon_candidates_kernel<WT>: one CTA per line, thread = lexicon entry.  The read is the pattern of the bit-parallel
// Levenshtein algorithm (Myers 1999, in Hyyro's global-distance block form): a per-line Peq table in shared memory, 64 classes x
// W = ceil(read_len / 64) words, and per entry id one lookup and about 15 integer operations per word.  The vertical deltas live
// in registers (WT >= W words, the template picks the smallest of 1, 2, 4, 8, 16).  The distance is read on the pattern's last
// row (the bit of row read_len - 1 in the last word), so the padding rows of the last word never matter.  An entry whose length
// differs from the read's by more than the cap is ruled out without work, and a column loop stops once the remaining ids
// cannot bring the distance back under the cap.
//   pass 1  distances up to the cap (max_edit, or the largest possible distance when max_edit < 0) -> a shared histogram
//           (integer atomics: the same counts in any order); warp 0 scans it for the cutoff distance D and how many entries to
//           take at D.
//   pass 2  the distances again, capped at D, in index order, 256 entries at a time; two block-wide prefix sums rank the
//           entries at D by index and place every taken entry in a shared list, which is therefore in index order.
//   order   rank of each listed entry by (distance, index), computed by counting: no sort network, no atomics, fixed bits.
// ctc_lexicon_score_kernel: one CTA per line.  The prologue writes the line's log2-softmax rows (x log2e - lse, the arithmetic of
// ctc.cu) for t < T_n into shared memory once, a warp per frame.  Then each warp scores one candidate at a time: the CTC alpha
// recursion (log2 domain, ctc.cu's lse3) with S = 2L+1 <= 127 states, 4 states per lane, the two states below a lane's first
// by shuffle, no CTA barrier per frame.  Every candidate of the line reads the same shared rows: the logits are read once.
#include "common.cuh"
#include <stdint.h>

namespace {

constexpr int LX_C = 64;
constexpr int LX_MAX_ENTRY = 63;             // S = 2L+1 <= 127: 4 states per lane of one warp
constexpr int LX_MAX_CAND = 256;
constexpr int LX_MAX_READ = 1024;            // read_stride: W <= 16 words of the pattern
constexpr int LX_MAX_T = 768;                // 256 B of log2-softmax per frame in shared memory
constexpr int LX_THREADS = 256;
constexpr int LX_WARPS = LX_THREADS / 32;
constexpr float LX_LOG2E = 1.4426950408889634f;
constexpr float LX_LN2 = 0.6931471805599453f;

typedef unsigned long long u64;

__device__ __forceinline__ bool lx_class(int c) { return c >= 0 && c < LX_C; }

// Levenshtein distance of the read (Peq [64][W], m ids, m >= 1) and the entry ent[0..n), or a value above `cap` once the
// distance is known to exceed it.
template <int WT>
__device__ __forceinline__ int lx_distance(const u64* __restrict__ peq, int W, int m, const int* __restrict__ ent, int n, int cap) {
  u64 pv[WT], mv[WT];
#pragma unroll
  for (int b = 0; b < WT; ++b) { pv[b] = ~0ull; mv[b] = 0ull; }
  const int rl = (m - 1) & 63;                            // the last pattern row inside word W-1
  int score = m;                                          // D[m][0]
  for (int j = 0; j < n; ++j) {
    const int c = __ldg(ent + j);
    const u64* eqrow = peq + (lx_class(c) ? c : 0) * W;
    const bool hit = lx_class(c);
    int hin = 1;                                          // D[0][j] - D[0][j-1] = 1: the global distance
#pragma unroll
    for (int b = 0; b < WT; ++b) {
      if (b >= W) break;
      // one 64-row block: hin is the horizontal delta entering above its first row, the result the one leaving below its last
      u64 eq = hit ? eqrow[b] : 0ull;
      const u64 neg = hin < 0 ? 1ull : 0ull, pos = hin > 0 ? 1ull : 0ull;
      const u64 xv = eq | mv[b];
      eq |= neg;
      const u64 xh = (((eq & pv[b]) + pv[b]) ^ pv[b]) | eq;
      u64 ph = mv[b] | ~(xh | pv[b]);
      u64 mh = pv[b] & xh;
      if (b == W - 1) score += (int)((ph >> rl) & 1ull) - (int)((mh >> rl) & 1ull);
      hin = (int)(ph >> 63) - (int)(mh >> 63);
      ph = (ph << 1) | pos;
      mh = (mh << 1) | neg;
      pv[b] = mh | ~(xv | ph);
      mv[b] = ph & xv;
    }
    if (score - (n - 1 - j) > cap) return cap + 1;       // each remaining column lowers D[m][.] by at most 1
  }
  return score;
}

// Block-wide exclusive prefix sum of v (every thread of the CTA calls it); *total gets the sum.  s_ws holds LX_WARPS + 1 ints.
__device__ __forceinline__ int lx_block_scan(int v, int* s_ws, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_ws[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = lane < LX_WARPS ? s_ws[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    if (lane < LX_WARPS) s_ws[lane + 1] = w;             // s_ws[k] = sum of warps below k
    if (lane == 0) s_ws[0] = 0;
  }
  __syncthreads();
  const int out = s_ws[warp] + x - v;
  *total = s_ws[LX_WARPS];
  __syncthreads();                                        // s_ws is free again
  return out;
}

template <int WT>
__global__ void __launch_bounds__(LX_THREADS)
lexicon_candidates_kernel(const int* __restrict__ reads, int read_stride, const int* __restrict__ read_len,
                          const int* __restrict__ lex_ids, const int* __restrict__ lex_off, int K, int max_entry_len, int max_edit,
                          int dmax, int max_cand, int* __restrict__ cand, int* __restrict__ cand_dist, int* __restrict__ cand_total) {
  __shared__ u64 s_peq[LX_C * WT];
  __shared__ int s_key[LX_MAX_CAND], s_idx[LX_MAX_CAND];
  __shared__ int s_ws[LX_WARPS + 1];
  __shared__ int s_cut, s_take, s_total;
  extern __shared__ int s_hist[];                         // [cap + 1]

  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int m = min(max(read_len[n], 0), read_stride);
  const int W = (m + 63) >> 6;
  const int* rd = reads + (size_t)n * read_stride;
  const int cap = max_edit < 0 ? dmax : min(max_edit, dmax);   // no distance exceeds dmax = max(read_stride, max_entry_len)

  // Peq[c][b]: bit i set where read id 64b + i equals c (ids outside [0, 64) set nothing: they match nothing)
  for (int i = tid; i < LX_C * W; i += LX_THREADS) {
    const int c = i / W, b = i - c * W;
    u64 w = 0ull;
    const int lo = 64 * b, hi = min(m, lo + 64);
    for (int p = lo; p < hi; ++p) w |= (u64)(__ldg(rd + p) == c) << (p - lo);
    s_peq[i] = w;
  }
  for (int i = tid; i <= cap; i += LX_THREADS) s_hist[i] = 0;
  __syncthreads();

  // distance of entry k, or a value above lim when it is larger than lim (or the entry is malformed)
  auto dist = [&](int k, int lim) {
    const int o = __ldg(lex_off + k), ln = __ldg(lex_off + k + 1) - o;
    if (ln < 0 || ln > max_entry_len || abs(ln - m) > lim) return lim + 1;
    if (m == 0) return ln;
    return lx_distance<WT>(s_peq, W, m, lex_ids + o, ln, lim);
  };

  // ---------------- pass 1: histogram of the distances within the cap ----------------
  for (int k0 = 0; k0 < K; k0 += LX_THREADS) {
    const int k = k0 + tid;
    if (k < K) {
      const int d = dist(k, cap);
      if (d <= cap) atomicAdd(s_hist + d, 1);
    }
  }
  __syncthreads();
  if (warp == 0) {                                        // cutoff: the smallest D with (entries at distance <= D) >= wanted
    int run = 0, cut = -1, take = 0;
    for (int d0 = 0; d0 <= cap; d0 += 32) {
      const int d = d0 + lane;
      int x = d <= cap ? s_hist[d] : 0;
      const int h = x;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      const int incl = run + x;
      if (cut < 0) {
        const unsigned hitm = __ballot_sync(0xffffffffu, d <= cap && h > 0 && incl >= max_cand);
        if (hitm) {
          const int src = __ffs(hitm) - 1;
          cut = d0 + src;
          take = max_cand - __shfl_sync(0xffffffffu, incl - h, src);
        }
      }
      run += __shfl_sync(0xffffffffu, x, 31);
    }
    if (lane == 0) {
      s_total = run;
      if (cut < 0) { cut = cap; take = run; }           // fewer than max_cand within the cap: all of them (take unused)
      s_cut = cut;
      s_take = take;
    }
  }
  __syncthreads();
  const int total = s_total, want = min(total, max_cand), cut = s_cut, take_at = s_take;

  // ---------------- pass 2: the taken entries in index order ----------------
  int seen_eq = 0, listed = 0;
  const bool all_within = total <= max_cand;
  for (int k0 = 0; k0 < K && listed < want; k0 += LX_THREADS) {
    const int k = k0 + tid;
    const int d = k < K ? dist(k, cut) : cut + 1;
    const bool lt = d < cut, eq = d == cut;
    if (!__syncthreads_or(lt || eq)) continue;
    int sel = lt || (eq && all_within);
    if (!all_within) {
      int neq;
      const int r = lx_block_scan(eq ? 1 : 0, s_ws, &neq);
      sel = lt || (eq && seen_eq + r < take_at);
      seen_eq += neq;
    }
    int nsel;
    const int p = lx_block_scan(sel, s_ws, &nsel);
    if (sel) { s_key[listed + p] = d; s_idx[listed + p] = k; }
    listed += nsel;
  }
  __syncthreads();

  // ---------------- order by (distance, index): the list is in index order ----------------
  int* oc = cand + (size_t)n * max_cand;
  int* od = cand_dist + (size_t)n * max_cand;
  for (int i = tid; i < max_cand; i += LX_THREADS) {
    if (i < want) {
      const int d = s_key[i];
      int r = 0;
      for (int j = 0; j < want; ++j) {
        const int dj = s_key[j];
        r += (dj < d) | (dj == d && j < i);
      }
      oc[r] = s_idx[i];
      od[r] = d;
    }
    if (i >= want) { oc[i] = -1; od[i] = -1; }
  }
  if (tid == 0) cand_total[n] = total;
}

// log2(2^a + 2^b + 2^c) with -inf handling (ctc.cu's lse3)
__device__ __forceinline__ float lx_lse3(float a, float b, float c) {
  const float m = fmaxf(a, fmaxf(b, c));
  if (m == -INFINITY) return -INFINITY;
  return m + ptx::lg2(ptx::ex2(a - m) + ptx::ex2(b - m) + ptx::ex2(c - m));
}

__device__ __forceinline__ float lx_pick(const float* a, int k) { return k == 0 ? a[0] : k == 1 ? a[1] : k == 2 ? a[2] : a[3]; }

__global__ void __launch_bounds__(LX_THREADS)
ctc_lexicon_score_kernel(const float* __restrict__ logits, const int* __restrict__ input_len, int T, int N, int blank,
                         const int* __restrict__ lex_ids, const int* __restrict__ lex_off, int max_entry_len,
                         const int* __restrict__ cand, int max_cand, float* __restrict__ score, int* __restrict__ best,
                         float* __restrict__ best_score) {
  extern __shared__ __align__(16) float s_lp[];          // [T_n][64] log2-softmax, then [max_cand] scores
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int Tn = max(0, min(input_len[n], T));
  float* s_sc = s_lp + (size_t)T * LX_C;

  // ---------------- prologue: warp = frame ----------------
  for (int t = warp; t < Tn; t += LX_WARPS) {
    const float* x = logits + ((size_t)t * N + n) * LX_C;
    const float x0 = __ldg(x + lane) * LX_LOG2E, x1 = __ldg(x + lane + 32) * LX_LOG2E;
    float m = fmaxf(x0, x1);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float sum = ptx::ex2(x0 - m) + ptx::ex2(x1 - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float lse = m + ptx::lg2(sum);
    s_lp[t * LX_C + lane] = x0 - lse;
    s_lp[t * LX_C + lane + 32] = x1 - lse;
  }
  __syncthreads();

  // ---------------- one candidate per warp at a time ----------------
  for (int j = warp; j < max_cand; j += LX_WARPS) {
    const int k = cand[(size_t)n * max_cand + j];
    float sc = -INFINITY;
    if (k >= 0) {
      const int o = __ldg(lex_off + k), L = __ldg(lex_off + k + 1) - o;
      if (L < 0 || L > max_entry_len) {
        sc = __int_as_float(0x7fc00000);
      } else {
        const int* ent = lex_ids + o;
        const int S = 2 * L + 1;
        int cls[4];
        bool skin[4];
        int bad = 0, rep = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int s = 4 * lane + q;
          cls[q] = blank;
          skin[q] = false;
          if (s < S && (s & 1)) {
            const int v = __ldg(ent + (s >> 1));
            if (v < 0 || v >= LX_C || v == blank) bad = 1;
            else cls[q] = v;
            if (s >= 3) {
              const bool same = v == __ldg(ent + (s >> 1) - 1);
              rep += same;
              skin[q] = !same;
            }
          }
        }
        if (__any_sync(0xffffffffu, bad)) {
          sc = __int_as_float(0x7fc00000);
        } else if (L + __reduce_add_sync(0xffffffffu, rep) > Tn) {
          sc = -INFINITY;                                 // infeasible (T_n = 0 with L = 0 is the empty path, score 0)
        } else if (Tn == 0) {
          sc = 0.f;
        } else {
          float a[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) a[q] = (4 * lane + q < 2 && 4 * lane + q < S) ? s_lp[cls[q]] : -INFINITY;
          for (int t = 1; t < Tn; ++t) {
            const float* row = s_lp + t * LX_C;
            float e[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) e[q] = row[cls[q]];
            float p2 = __shfl_up_sync(0xffffffffu, a[2], 1), p1 = __shfl_up_sync(0xffffffffu, a[3], 1);
            if (lane == 0) { p2 = -INFINITY; p1 = -INFINITY; }
            const float v[6] = {p2, p1, a[0], a[1], a[2], a[3]};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float nv = lx_lse3(v[q + 2], v[q + 1], skin[q] ? v[q] : -INFINITY) + e[q];
              a[q] = (4 * lane + q < S) ? nv : -INFINITY;
            }
          }
          const float v1 = __shfl_sync(0xffffffffu, lx_pick(a, (S - 1) & 3), (S - 1) >> 2);
          const float v2 = S >= 2 ? __shfl_sync(0xffffffffu, lx_pick(a, (S - 2) & 3), (S - 2) >> 2) : -INFINITY;
          sc = lx_lse3(v1, v2, -INFINITY) * LX_LN2;
        }
      }
    }
    if (lane == 0) {
      score[(size_t)n * max_cand + j] = sc;
      s_sc[j] = sc;
    }
  }
  __syncthreads();

  // ---------------- the highest finite score, lowest slot on ties ----------------
  if (warp == 0) {
    float bv = -INFINITY;
    int bj = -1;
    for (int j = lane; j < max_cand; j += 32) {
      const float v = s_sc[j];
      if (isfinite(v) && (bj < 0 || v > bv)) { bv = v; bj = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (oj >= 0 && (bj < 0 || ov > bv || (ov == bv && oj < bj))) { bv = ov; bj = oj; }
    }
    if (lane == 0) {
      best[n] = bj >= 0 ? cand[(size_t)n * max_cand + bj] : -1;
      best_score[n] = bj >= 0 ? bv : -INFINITY;
    }
  }
}

}  // namespace

extern "C" int crnn_lexicon_candidates(const int* reads, int read_stride, const int* read_len, int N, const int* lex_ids,
                                       const int* lex_off, int K, int max_entry_len, int max_edit, int max_candidates, int* cand,
                                       int* cand_dist, int* cand_total, crnn_stream_t stream) {
  if (!reads || !read_len || !lex_ids || !lex_off || !cand || !cand_dist || !cand_total)
    return crnn_fail(CRNN_INVALID_VALUE, "lexicon_candidates: null pointer");
  if (N <= 0 || K <= 0 || read_stride < 0 || max_entry_len < 0 || max_candidates < 1 || max_candidates > LX_MAX_CAND)
    return crnn_fail(CRNN_INVALID_VALUE, "lexicon_candidates: bad shape (N = %d, K = %d, read_stride = %d, max_entry_len = %d, "
                     "max_candidates = %d, which must lie in [1, %d])", N, K, read_stride, max_entry_len, max_candidates, LX_MAX_CAND);
  if (max_entry_len > LX_MAX_ENTRY)
    return crnn_fail(CRNN_UNSUPPORTED, "lexicon_candidates: max_entry_len = %d is beyond the kernel (<= %d)", max_entry_len, LX_MAX_ENTRY);
  if (read_stride > LX_MAX_READ)
    return crnn_fail(CRNN_UNSUPPORTED, "lexicon_candidates: read_stride = %d is beyond the kernel (<= %d)", read_stride, LX_MAX_READ);
  const int dmax = max(read_stride, max_entry_len);
  const int cap = max_edit < 0 ? dmax : min(max_edit, dmax);
  const size_t smem = sizeof(int) * (size_t)(cap + 1);
  const int words = (read_stride + 63) / 64;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define LX_LAUNCH(WT)                                                                                                         \
  lexicon_candidates_kernel<WT><<<N, LX_THREADS, smem, st>>>(reads, read_stride, read_len, lex_ids, lex_off, K, max_entry_len, \
                                                             max_edit, dmax, max_candidates, cand, cand_dist, cand_total)
  if (words <= 1) LX_LAUNCH(1);
  else if (words <= 2) LX_LAUNCH(2);
  else if (words <= 4) LX_LAUNCH(4);
  else if (words <= 8) LX_LAUNCH(8);
  else LX_LAUNCH(16);
#undef LX_LAUNCH
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}

extern "C" int crnn_ctc_lexicon_score(const float* logits, const int* input_len, int T, int N, int C, int blank, const int* lex_ids,
                                      const int* lex_off, int max_entry_len, const int* cand, int max_candidates, float* score,
                                      int* best, float* best_score, crnn_stream_t stream) {
  if (!logits || !input_len || !lex_ids || !lex_off || !cand || !score || !best || !best_score)
    return crnn_fail(CRNN_INVALID_VALUE, "ctc_lexicon_score: null pointer");
  if (T <= 0 || N <= 0 || max_entry_len < 0 || max_candidates < 1 || max_candidates > LX_MAX_CAND)
    return crnn_fail(CRNN_INVALID_VALUE, "ctc_lexicon_score: bad shape (T = %d, N = %d, max_entry_len = %d, max_candidates = %d, "
                     "which must lie in [1, %d])", T, N, max_entry_len, max_candidates, LX_MAX_CAND);
  if (C != LX_C) return crnn_fail(CRNN_UNSUPPORTED, "ctc_lexicon_score: C must be 64, got %d", C);
  if (blank < 0 || blank >= C) return crnn_fail(CRNN_INVALID_VALUE, "ctc_lexicon_score: blank %d outside [0, %d)", blank, C);
  if (T > LX_MAX_T)
    return crnn_fail(CRNN_UNSUPPORTED, "ctc_lexicon_score: T = %d is beyond the kernel (<= %d frames in shared memory)", T, LX_MAX_T);
  if (max_entry_len > LX_MAX_ENTRY)
    return crnn_fail(CRNN_UNSUPPORTED, "ctc_lexicon_score: max_entry_len = %d is beyond the kernel (<= %d)", max_entry_len, LX_MAX_ENTRY);
  const size_t smem = sizeof(float) * ((size_t)T * LX_C + max_candidates);
  if (smem > 48 * 1024)
    CUDA_TRY(cudaFuncSetAttribute(ctc_lexicon_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ctc_lexicon_score_kernel<<<N, LX_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      logits, input_len, T, N, blank, lex_ids, lex_off, max_entry_len, cand, max_candidates, score, best, best_score);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
