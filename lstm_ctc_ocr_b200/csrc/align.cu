// CTC forced alignment (Viterbi) for C = 64 classes, sm_90a: the best path of a given labelling, each label's frame span and
// its peak posterior.  The max-plus form of the alpha recursion of csrc/ctc.cu, followed by a backtrace.
//
// ctc_align_kernel: one CTA per utterance, 4 consecutive states per thread (ctc_long_kernel's layout), CTA size from
// max_label_len at launch (32 .. 320 threads, S_pad = 2L+1 rounded up to 4 <= 1280).  The caller's workspace holds, per
// utterance, the log-softmax normaliser of every frame, the backtraced path and one predecessor byte per (frame, state).
//   prologue   warp = frame, 8 frames' loads in flight per warp: lse_t = m + log(sum exp(x - m)) of the 64-float row -> workspace
//   recursion  v_t(s) = e_t(s) + max(v_{t-1}(s), v_{t-1}(s-1), v_{t-1}(s-2) where the skip is allowed), natural log; the
//              previous row ping-pongs in shared memory (one barrier per frame), the choice (0, 1, 2 = states stepped back) is
//              stored as 4 bytes per thread.  Emissions e = x - lse are loaded four frames ahead: the chain is max + add only.
//              Ties: s beats s-1 beats s-2 (strict comparisons in that order); at the end S-1 beats S-2.
//   backtrace  32 frames per round: the CTA loads the 32 x 68 bytes of choices the path can reach (the state falls by at
//              most 2 per frame) into shared memory, one thread walks them; the path goes to the workspace.
//   spans      thread = frame: a label state's first / last frame writes start / end; peak = max over the span of
//              exp(x - lse) through an integer atomicMax on the float bits (non-negative floats order as their bits), so the
//              result is the same bits run to run.
// Logits are read one float at a time (4-byte alignment is enough).  No tensor cores: the dynamic program is a scan.
#include "common.cuh"
#include <limits.h>
#include <stdint.h>

namespace {

constexpr int AL_C = 64;
constexpr int AL_MAX_LABEL = 639;
constexpr int AL_MAX_THREADS = 320;
constexpr int AL_WS_ALIGN = 256;     // the launch rounds the workspace pointer up to this; the size query includes it
constexpr int BT_ROWS = 32;          // frames per backtrace round
constexpr int BT_WORDS = 17;         // 68 bytes of choices per frame: states lo .. lo+67 with lo = (s - 63) & ~3 cover s-62 .. s
constexpr int PRO_RB = 8;            // prologue rows per warp per batch: all their loads are issued before any use
constexpr int EM_AHEAD = 4;          // emissions loaded this many frames ahead of the recursion step that uses them

__host__ __device__ inline int al_stride(int max_label_len) { return (2 * max_label_len + 1 + 3) & ~3; }   // S_pad, a multiple of 4

__device__ __forceinline__ float al_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float al_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(AL_MAX_THREADS, 3)   // 3 CTAs of 320 threads per SM: 300 long lines in one wave
ctc_align_kernel(const float* __restrict__ logits, const int* __restrict__ labels, int label_stride, const int* __restrict__ label_len,
                 const int* __restrict__ input_len, int T, int N, int blank, int max_label_len, int* __restrict__ start,
                 int* __restrict__ end, float* __restrict__ peak, float* __restrict__ path_logprob, float* ws) {
  extern __shared__ __align__(16) float asm_[];
  const int AS = al_stride(max_label_len);
  const int BS = AS + 8;                                  // a row: 4 pad, AS states, 4 pad (pads stay -inf)
  float* s_buf = asm_;                                    // [2][BS]
  int* s_ext = reinterpret_cast<int*>(s_buf + 2 * BS);    // [AS] class of each state (blank past S)
  int* s_peak = s_ext + AS;                               // [max(1, max_label_len)] float bits of each label's peak
  uint32_t* s_win = reinterpret_cast<uint32_t*>(s_peak + (max_label_len > 0 ? max_label_len : 1));   // [BT_ROWS][BT_WORDS]
  __shared__ int s_off, s_repeats, s_bad, s_st;

  const int n = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int warp = tid >> 5, lane = tid & 31, nw = nt >> 5;
  const bool dense = label_stride > 0;
  const int L = label_len[n];
  const int Tn = max(0, min(input_len[n], T));
  const int S = 2 * L + 1;
  float* lse = ws + (size_t)n * T;                                                        // [T] normaliser
  int* path = reinterpret_cast<int*>(ws + (size_t)N * T) + (size_t)n * T;                 // [T] state of each frame
  uint32_t* bp = reinterpret_cast<uint32_t*>(ws + (size_t)2 * N * T) + (size_t)n * T * (AS / 4);   // [T][AS] bytes

  if (warp == 0) {
    int acc = 0;
    if (!dense)
      for (int i = lane; i < n; i += 32) acc += __ldg(label_len + i);
    acc = __reduce_add_sync(0xffffffffu, acc);
    if (lane == 0) { s_off = dense ? 0 : acc; s_repeats = 0; s_bad = 0; }
  }
  __syncthreads();
  const size_t base = dense ? (size_t)n * label_stride : (size_t)s_off;
  const int* lab = labels + base;
  bool too_long = L < 0 || L > max_label_len || (dense && L > label_stride);
  if (!too_long) {
    int rep = 0, bad = 0;
    for (int s = tid; s < AS; s += nt) {
      int v = blank;
      if (s < S && (s & 1)) {
        v = lab[s >> 1];
        // ids outside [0,C) or equal to the blank are never used as indices: the utterance is rejected (NaN)
        if (v < 0 || v >= AL_C || v == blank) { bad = 1; v = blank; }
        if (s >= 3 && v == lab[(s >> 1) - 1]) rep++;
      }
      s_ext[s] = v;
    }
    for (int k = tid; k < L; k += nt) s_peak[k] = 0;
    if (rep) atomicAdd(&s_repeats, rep);
    if (bad) atomicOr(&s_bad, 1);
  }
  __syncthreads();
  too_long = too_long || s_bad != 0;
  // entries this call owns: a dense row in full (padding past L included), else the utterance's L flat entries
  const int owned = dense ? label_stride : max(L, 0);
  const bool feasible = !too_long && L + s_repeats <= Tn;
  if (!feasible) {
    for (int k = tid; k < owned; k += nt) { start[base + k] = -1; end[base + k] = -1; peak[base + k] = 0.f; }
    if (tid == 0) path_logprob[n] = too_long ? __int_as_float(0x7fc00000) : -INFINITY;
    return;
  }
  for (int k = L + tid; k < owned; k += nt) { start[base + k] = -1; end[base + k] = -1; peak[base + k] = 0.f; }
  if (Tn == 0) {                                          // L = 0 here: the empty path
    if (tid == 0) path_logprob[n] = 0.f;
    return;
  }

  // ---------------- prologue: warp = frame, normalisers to the workspace ----------------
  for (int t0 = warp; t0 < Tn; t0 += PRO_RB * nw) {
    float x0[PRO_RB], x1[PRO_RB], m[PRO_RB], sum[PRO_RB];
#pragma unroll
    for (int u = 0; u < PRO_RB; ++u) {
      const int t = min(t0 + u * nw, Tn - 1);
      const float* x = logits + ((size_t)t * N + n) * AL_C;
      x0[u] = __ldg(x + lane);
      x1[u] = __ldg(x + lane + 32);
    }
#pragma unroll
    for (int u = 0; u < PRO_RB; ++u) m[u] = fmaxf(x0[u], x1[u]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
      for (int u = 0; u < PRO_RB; ++u) m[u] = fmaxf(m[u], __shfl_xor_sync(0xffffffffu, m[u], o));
#pragma unroll
    for (int u = 0; u < PRO_RB; ++u) sum[u] = expf(x0[u] - m[u]) + expf(x1[u] - m[u]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
      for (int u = 0; u < PRO_RB; ++u) sum[u] += __shfl_xor_sync(0xffffffffu, sum[u], o);
#pragma unroll
    for (int u = 0; u < PRO_RB; ++u) {
      const int t = t0 + u * nw;
      if (lane == 0 && t < Tn) lse[t] = m[u] + logf(sum[u]);
    }
  }
  for (int i = tid; i < 2 * BS; i += nt) s_buf[i] = -INFINITY;
  __syncthreads();

  const int s0 = 4 * tid;                                 // this thread's states s0 .. s0+3 (none when s0 >= AS)
  const bool act = s0 < AS;
  int cls[4];
  bool skin[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int s = s0 + k;
    cls[k] = act ? s_ext[s] : blank;
    skin[k] = act && s >= 2 && s < S && s_ext[s] != blank && s_ext[s] != s_ext[s - 2];
  }
  auto emit = [&](int t, float* e) {
    const float* x = logits + ((size_t)t * N + n) * AL_C;
    const float l = lse[t];
#pragma unroll
    for (int k = 0; k < 4; ++k) e[k] = __ldg(x + cls[k]) - l;
  };

  // ---------------- max-plus recursion ----------------
  float a[4], ep[EM_AHEAD][4];                            // ep[j]: emissions of frame t+j at step t
  if (act) {
    float e0[4];
    emit(0, e0);
#pragma unroll
    for (int k = 0; k < 4; ++k) a[k] = (s0 + k < 2 && s0 + k < S) ? e0[k] : -INFINITY;
    *reinterpret_cast<float4*>(s_buf + 4 + s0) = make_float4(a[0], a[1], a[2], a[3]);
#pragma unroll
    for (int j = 0; j < EM_AHEAD; ++j) {
      if (1 + j < Tn) emit(1 + j, ep[j]);
      else for (int k = 0; k < 4; ++k) ep[j][k] = 0.f;
    }
  }
  __syncthreads();
  for (int t = 1; t < Tn; ++t) {
    if (act) {
      const float* prev = s_buf + ((t - 1) & 1) * BS;
      float* cur = s_buf + (t & 1) * BS;
      float e[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) e[k] = ep[0][k];
#pragma unroll
      for (int j = 0; j + 1 < EM_AHEAD; ++j)
#pragma unroll
        for (int k = 0; k < 4; ++k) ep[j][k] = ep[j + 1][k];
      if (t + EM_AHEAD < Tn) emit(t + EM_AHEAD, ep[EM_AHEAD - 1]);
      const float2 lo = *reinterpret_cast<const float2*>(prev + 4 + s0 - 2);     // states s0-2, s0-1
      const float v[6] = {lo.x, lo.y, a[0], a[1], a[2], a[3]};
      uint32_t choice = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float best = v[k + 2];
        uint32_t c = 0;
        if (v[k + 1] > best) { best = v[k + 1]; c = 1; }
        if (skin[k] && v[k] > best) { best = v[k]; c = 2; }
        a[k] = (s0 + k < S) ? best + e[k] : -INFINITY;
        choice |= c << (8 * k);
      }
      *reinterpret_cast<float4*>(cur + 4 + s0) = make_float4(a[0], a[1], a[2], a[3]);
      bp[(size_t)t * (AS / 4) + tid] = choice;
    }
    __syncthreads();
  }

  const float* last = s_buf + ((Tn - 1) & 1) * BS + 4;
  const float v1 = last[S - 1], v2 = S >= 2 ? last[S - 2] : -INFINITY;
  const bool from2 = v2 > v1;
  const float best = from2 ? v2 : v1;
  if (tid == 0) path_logprob[n] = best;
  if (!(best > -INFINITY)) {                              // no path with a finite score (non-finite logits): no spans
    for (int k = tid; k < L; k += nt) { start[base + k] = -1; end[base + k] = -1; peak[base + k] = 0.f; }
    return;
  }
  if (L == 0) return;

  // ---------------- backtrace ----------------
  if (tid == 0) {
    s_st = from2 ? S - 2 : S - 1;
    path[Tn - 1] = s_st;
  }
  __syncthreads();
  const uint8_t* win = reinterpret_cast<const uint8_t*>(s_win);
  for (int t1 = Tn - 1; t1 > 0; t1 -= BT_ROWS) {
    const int st = s_st;
    const int lo = max(0, st - (2 * BT_ROWS - 1)) & ~3;
    const int rows = min(BT_ROWS, t1);
    for (int i = tid; i < rows * BT_WORDS; i += nt) {
      const int r = i / BT_WORDS, w = i - r * BT_WORDS;
      const int s = lo + 4 * w;
      s_win[i] = s < AS ? bp[(size_t)(t1 - r) * (AS / 4) + (s >> 2)] : 0u;
    }
    __syncthreads();
    if (tid == 0) {
      int s = st;
      for (int r = 0; r < rows; ++r) {
        s -= win[r * (4 * BT_WORDS) + (s - lo)];
        path[t1 - r - 1] = s;
      }
      s_st = s;
    }
    __syncthreads();
  }

  // ---------------- spans and peaks ----------------
  for (int t = tid; t < Tn; t += nt) {
    const int st = path[t];
    if (st & 1) {
      const int k = st >> 1;
      if (t == 0 || path[t - 1] != st) start[base + k] = t;
      if (t == Tn - 1 || path[t + 1] != st) end[base + k] = t + 1;
      const float y = expf(__ldg(logits + ((size_t)t * N + n) * AL_C + s_ext[st]) - lse[t]);
      atomicMax(s_peak + k, __float_as_int(y));
    }
  }
  __syncthreads();
  for (int k = tid; k < L; k += nt) peak[base + k] = __int_as_float(s_peak[k]);
}

// Workspace of ctc_align_kernel: per utterance T normalisers (f32), T path states (i32) and T rows of S_pad choice bytes, plus
// the alignment slack.  No crnn_fail here.
int align_bytes(int T, int N, int max_label_len, size_t* bytes) {
  if (max_label_len > AL_MAX_LABEL) return CRNN_UNSUPPORTED;
  const size_t per = (size_t)T * (size_t)(8 + al_stride(max_label_len));
  if (per > (SIZE_MAX - AL_WS_ALIGN) / (size_t)N) return CRNN_UNSUPPORTED;
  *bytes = per * (size_t)N + AL_WS_ALIGN;
  return CRNN_OK;
}

}  // namespace

extern "C" int crnn_ctc_align_workspace_size(int T, int N, int C, int max_label_len, size_t* bytes) {
  if (!bytes || T <= 0 || N <= 0 || max_label_len < 0) return crnn_fail(CRNN_INVALID_VALUE, "ctc_align_workspace_size: bad args");
  if (C != AL_C) return crnn_fail(CRNN_UNSUPPORTED, "ctc_align: C must be 64");
  if (align_bytes(T, N, max_label_len, bytes) != CRNN_OK)
    return crnn_fail(CRNN_UNSUPPORTED, "ctc_align: max_label_len = %d, T = %d, N = %d is beyond the kernel (max_label_len <= %d, "
                     "size within size_t)", max_label_len, T, N, AL_MAX_LABEL);
  return CRNN_OK;
}

extern "C" int crnn_ctc_align(const float* logits, const int* labels, int label_stride, const int* label_len, const int* input_len,
                              int T, int N, int C, int blank, int max_label_len, int* start, int* end, float* peak,
                              float* path_logprob, void* workspace, size_t workspace_bytes, crnn_stream_t stream) {
  if (!logits || !labels || !label_len || !input_len || !start || !end || !peak || !path_logprob || !workspace)
    return crnn_fail(CRNN_INVALID_VALUE, "ctc_align: null pointer");
  if (T <= 0 || N <= 0 || max_label_len < 0 || label_stride < 0) return crnn_fail(CRNN_INVALID_VALUE, "ctc_align: bad shape");
  if (C != AL_C) return crnn_fail(CRNN_UNSUPPORTED, "ctc_align: C must be 64");
  if (blank < 0 || blank >= C) return crnn_fail(CRNN_INVALID_VALUE, "ctc_align: blank %d outside [0, %d)", blank, C);
  size_t need = 0;
  if (align_bytes(T, N, max_label_len, &need) != CRNN_OK)
    return crnn_fail(CRNN_UNSUPPORTED, "ctc_align: max_label_len = %d is beyond the kernel (<= %d) or the workspace overflows",
                     max_label_len, AL_MAX_LABEL);
  if (workspace_bytes < need)
    return crnn_fail(CRNN_WORKSPACE_TOO_SMALL, "ctc_align: the workspace needs %zu bytes, got %zu", need, workspace_bytes);
  float* ws = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(workspace) + AL_WS_ALIGN - 1) & ~uintptr_t(AL_WS_ALIGN - 1));
  const int AS = al_stride(max_label_len);
  const int threads = min(AL_MAX_THREADS, (AS / 4 + 31) / 32 * 32);
  const size_t smem = sizeof(float) * 2 * (AS + 8) + sizeof(int) * (AS + (max_label_len > 0 ? max_label_len : 1)) +
                      sizeof(uint32_t) * BT_ROWS * BT_WORDS;
  ctc_align_kernel<<<N, threads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      logits, labels, label_stride, label_len, input_len, T, N, blank, max_label_len, start, end, peak, path_logprob, ws);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
