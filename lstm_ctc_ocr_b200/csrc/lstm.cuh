// Persistent BiLSTM recurrence for sm_90a: one thread-block CLUSTER per (direction, 128-sample batch tile).
//
// Replaces the tf.while_loop of tf.contrib.rnn.LSTMCell(256) under bidirectional_dynamic_rnn
// (lib/networks/network.py:104-107): per step  z = x_t W_x + b (precomputed, `xproj`) + h_{t-1} W_h ;
// i,j,f,o = split(z); c = sigma(f+1) c + sigma(i) tanh(j); h = sigma(o) tanh(c); zero output past sequence_length.
//
// lstm_mc_kernel<CS>: two independent 64-row half pipelines per CTA; the cell runs on the wgmma accumulator fragments, h is
// exchanged as 4 KB half slices that land directly in every CTA's no-swizzle A operand, signalled through mbarriers; no cluster
// barrier per step (details above the kernel).
// Clusters are independent (no grid-wide sync), so partial residency cannot deadlock.
// The backward direction reads xproj rows that the projection GEMM already stored reversed-by-length, so both
// directions index step s uniformly; outputs are written back at t = len-1-s.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace lstm {

constexpr int BLOCK_M = 128;
constexpr int MC_THREADS = 128 + 8 * 32;   // warpgroup 0 setup, warps 4.. MMA + cell (two warpgroups, one per half)

struct Params {
  const __nv_bfloat16* xproj;   // [Nimg*H, 2048]: [fw 1024 | bw 1024 (rows reversed by length)], permuted columns
  __nv_bfloat16* h_state;       // [2 bufs][2 dirs][Npad][256]
  __nv_bfloat16* lstm_out;      // [Nimg*H, 512]
  const int* seq_len;           // [Nimg]
  int Nimg, Npad, H, T, tiles_per_dir;
  // training only (nullptr for inference): activations the backward recurrence needs
  __nv_bfloat16* gates;         // post-activation gates i,j,f,o, coalesced per batch tile: layout in common.cuh (lstm_gate_off)
  float* csave;                 // cell state after the step (lstm_c_off)
  long long* trace;             // debug (CRNN_LSTM_TRACE=1): clock64 stamps [CTA 0 / 5][warpgroup slot 0 / 1][steps 8..11][16 events]
};

// debug timeline: one stamp per (selected CTA, warpgroup slot, step, event); all stamps of a CTA come from the same SM clock
#define LSTM_TRACE_WG(wg, ev)                                                                           \
  do {                                                                                                  \
    if (p.trace != nullptr && lane == 0 && s >= 8 && s < 12 && (blockIdx.x == 0 || blockIdx.x == 5))    \
      p.trace[((((blockIdx.x ? 1 : 0) * 2 + (wg)) * 4 + (s - 8)) * 16) + (ev)] = clock64();             \
  } while (0)

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_arrive_release() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait_acquire() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------------------------------------
// The recurrence without a cluster barrier (and without fence.proxy.async + a 64 KB TMA fetch of h per CTA) on the per-step
// critical path (CRNN_LSTM_TRACE=1 prints the clock64 timeline of a few steps):
//
//   * rows of a batch tile never interact, so the two MMA warpgroups run two INDEPENDENT recurrences, warpgroup `wgi` over rows
//     64*wgi .. 64*wgi+63 (a "half"): each half has its own A buffers, mbarriers, named barrier and exchange, and never waits
//     for the other half's rows (in practice the halves stay close to lockstep: their peers deliver both at about the same time)
//   * the A operand (h_{t-1}) lives in shared memory WITHOUT swizzle, half-major as [2 halves][32 K-chunks][64 rows][16 B]
//     (8-row x 16-B core matrices, LBO = 1024, SBO = 128), so the 32 units one CTA produces for one half are ONE contiguous
//     4 KB slice
//   * the cell runs on the wgmma accumulator fragment itself (wgmma.cuh): with the columns of Bh ordered [i|j|f|o] x 32 units,
//     a thread's m64n128 fragment holds all four gates of units 8k + 2(l%4) + {0,1} (k = 0..3) for rows 16w + l/4 and +8;
//     the cell state of those 16 cells stays in registers for all T steps.  No accumulator staging, no barrier before the cell.
//   * each thread stores its h_t words (bf16 pairs) straight into this CTA's own copy of the next A buffer (st.shared); one
//     lane then bulk-stores the slice to global memory (L2) and, once written, multicasts it from there into the 7 peers' A
//     buffers, crediting THEIR mbarriers: no generic-proxy global stores, hence no full fence.proxy.async on the critical path
//   * the MMA warpgroup of each half waits on its own mbarrier (8 slices) and goes; nobody waits for a cluster barrier
//   * A is double buffered: a slice of h_t can only be sent after its sender saw h_{t-1} from every CTA, i.e. after every CTA's
//     MMA of step t-1 of the same half (the last reader of that buffer) has completed -- causality replaces a "buffer free"
//     handshake.  A half runs and exchanges all T steps even when none of its rows is valid: its peers wait for its slices.
// Global exchange buffer: p.h_state viewed as [2 bufs][2*tiles_per_dir units][2 halves][8 ranks][4 KB].

template <int CS>
struct CfgMc {
  static constexpr int UPC = 256 / CS;
  static constexpr int NCOLS = 4 * UPC;
  static constexpr int B_BYTES = 4 * NCOLS * 128;         // resident W_h slice (SW128 K-major, 4 K-blocks of 64)
  static constexpr int HALF_ROWS = BLOCK_M / 2;           // rows of one half (one MMA warpgroup)
  static constexpr int HALF_A_BYTES = 32 * HALF_ROWS * 16;  // [32 K-chunks][64 rows][16 B] = 32 KB
  static constexpr int A_BYTES = 2 * HALF_A_BYTES;        // one A buffer, both halves: 64 KB
  static constexpr int SLICE_BYTES = HALF_A_BYTES / CS;   // 4 KB: the 4 K-chunks one CTA produces for one half
  static constexpr int BAR_OFFSET = 2 * A_BYTES + B_BYTES;
  static constexpr int SMEM_BYTES = BAR_OFFSET + 128 + 1024;
};

template <int CS>
__global__ void __launch_bounds__(MC_THREADS, 1)
lstm_mc_kernel(const __grid_constant__ CUtensorMap tmW, const Params p) {
  static_assert(CS == 8, "8 CTAs x 32 units");
  using C = CfgMc<CS>;
  constexpr int UPC = C::UPC, NCOLS = C::NCOLS;
  static_assert(NCOLS == 128, "fragment column group j = gate j/4, units 8(j%4) ..: one m64n128 product per half and step");
  constexpr uint32_t FILL_TX = (CS - 1) * C::SLICE_BYTES;     // the 7 peers' slices; the own slice is written in place

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);   // offset arithmetic keeps the shared address space (STS)
  uint8_t* smem_a = smem;                                   // [2 bufs][2 halves][HALF_A_BYTES]
  uint8_t* smem_b = smem + 2 * C::A_BYTES;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + C::BAR_OFFSET);   // [2 halves][2 bufs]
  uint64_t* b_full = a_full + 4;

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = (int)cluster_ctarank();
  const int unit = blockIdx.x / CS;                   // (dir, batch tile)
  const int dir = unit / p.tiles_per_dir;
  const int tile = unit - dir * p.tiles_per_dir;

  if (warp_idx == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmW);
    // one arrival arms the byte count (MMA warpgroup), the other says "the local slice is in place" (exchange lane)
    for (int i = 0; i < 4; ++i) ptx::mbar_init(&a_full[i], 2);
    ptx::mbar_init(b_full, 1);
    ptx::fence_barrier_init();
    // first fills of each half: buffer 1 receives h_0 (consumed at step 1), buffer 0 receives h_1 (consumed at step 2)
    for (int hf = 0; hf < 2; ++hf) {
      if (p.T > 1) ptx::mbar_arrive_expect_tx(&a_full[2 * hf + 1], FILL_TX);
      if (p.T > 2) ptx::mbar_arrive_expect_tx(&a_full[2 * hf + 0], FILL_TX);
    }
    ptx::mbar_arrive_expect_tx(b_full, C::B_BYTES);
    for (int kb = 0; kb < 4; ++kb)
      ptx::tma_load_2d(&tmW, b_full, smem_b + kb * NCOLS * 128, kb * 64, dir * 1024 + rank * NCOLS);
  }
  __syncthreads();
  // peers write into this CTA's smem and credit its mbarriers: everything above must be in place cluster-wide first
  cluster_arrive_release();
  cluster_wait_acquire();

  if (warp_idx < 4) {
    ptx::setmaxnreg_dec<40>();
  } else {
    // ===================== one half per MMA warpgroup: MMA + cell on the accumulator fragment, cell state in registers
    ptx::setmaxnreg_inc<232>();
    const int wgi = (warp_idx >> 2) - 1;              // half: rows 64*wgi .. of the batch tile
    const int w = warp_idx & 3, q4 = lane & 3;
    const int rr0 = 16 * w + (lane >> 2);             // fragment rows rr0 and rr0 + 8 of the half
    int n[2], len[2];
    bool okn[2];
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      n[rh] = tile * BLOCK_M + wgi * C::HALF_ROWS + rr0 + 8 * rh;
      okn[rh] = n[rh] < p.Nimg;
      len[rh] = okn[rh] ? min(max(__ldg(p.seq_len + n[rh]), 0), p.T) : 0;
    }
    float cst[2][4][2];                               // [row][k][unit 8k + 2*q4 + e]
#pragma unroll
    for (int rh = 0; rh < 2; ++rh)
#pragma unroll
      for (int k = 0; k < 4; ++k) { cst[rh][k][0] = 0.f; cst[rh][k][1] = 0.f; }
    uint64_t* my_full = a_full + 2 * wgi;
    ptx::mbar_wait(b_full, 0);
    // this thread's 4-byte h words inside a half slice: K-chunk k (units 8k ..) at k*1024, row at 16 B per row, + 4 B per lane pair
    const uint32_t word_off = rr0 * 16 + q4 * 4;
    uint8_t* hx_half = reinterpret_cast<uint8_t*>(p.h_state) + (size_t)(unit * 2 + wgi) * C::HALF_A_BYTES;
    const size_t hx_buf_stride = (size_t)2 * p.tiles_per_dir * C::A_BYTES;

    for (int s = 0; s < p.T; ++s) {
      bool active[2];
      int t[2];
      // this step's input projection (row n, step s; bw rows were stored reversed by the projection GEMM): [row][gate][k] bf16 pairs,
      // issued before the h wait so that the loads are in flight during it
      uint32_t xw[2][4][4];
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        active[rh] = s < len[rh];
        t[rh] = active[rh] ? (dir ? (len[rh] - 1 - s) : s) : s;
        if (active[rh]) {
          const uint32_t* src = reinterpret_cast<const uint32_t*>(p.xproj + ((size_t)n[rh] * p.H + s) * 2048 + dir * 1024 + rank * NCOLS + 2 * q4);
#pragma unroll
          for (int g = 0; g < 4; ++g)
#pragma unroll
            for (int k = 0; k < 4; ++k) xw[rh][g][k] = __ldg(src + (g * UPC + 8 * k) / 2);
        } else {
#pragma unroll
          for (int g = 0; g < 4; ++g)
#pragma unroll
            for (int k = 0; k < 4; ++k) xw[rh][g][k] = 0u;
        }
      }
      // the next step's 2 x 128-B lines of the same rows into L2: xproj (268 MB at the benchmark shape) comes from HBM, and a
      // miss there would otherwise surface in the cell of the next step (the loads above have one h wait to land, not more)
      if (q4 < 2) {
#pragma unroll
        for (int rh = 0; rh < 2; ++rh)
          if (s + 1 < len[rh])
            asm volatile("prefetch.global.L2 [%0];" ::"l"(p.xproj + ((size_t)n[rh] * p.H + s + 1) * 2048 + dir * 1024 + rank * NCOLS + q4 * 64));
      }
      if (w == 0) LSTM_TRACE_WG(wgi, 5);
      float d[NCOLS / 2];
      if (s > 0) {
        const int b = s & 1;
        ptx::mbar_wait(&my_full[b], ((s - 1) >> 1) & 1);
        if (w == 0) LSTM_TRACE_WG(wgi, 3);
        // next fill of this buffer is h_{s+1}, consumed at step s+2; its senders are all behind this wait (see header)
        if (s + 2 < p.T && (threadIdx.x & 127) == 0) ptx::mbar_arrive_expect_tx(&my_full[b], FILL_TX);
        const uint32_t a_base = ptx::smem_u32(smem_a + b * C::A_BYTES + wgi * C::HALF_A_BYTES);
        wg::fence();
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          const uint64_t a_desc = ptx::make_desc_k_nosw(a_base + k * 2048, 1024, 128);
          const uint64_t b_desc = ptx::make_desc_k_sw128(ptx::smem_u32(smem_b + (k >> 2) * NCOLS * 128)) + 2 * (k & 3);
          wg::mma_bf16<NCOLS>(d, a_desc, b_desc, k != 0);
        }
        wg::commit();
        wg::wait<0>();
        wg::fence_operand(d);
        if (w == 0) LSTM_TRACE_WG(wgi, 4);
      } else {
#pragma unroll
        for (int i = 0; i < NCOLS / 2; ++i) d[i] = 0.f;
      }
      // ---- the cell on the fragment: gate g of (row rh, unit 8k + 2*q4 + e) is d[16g + 4k + 2rh + e]; the activations overwrite
      // the (then dead) pre-activations for the saved training state
      uint32_t hw[2][4];                              // h_t as bf16 pairs [row][k]
#pragma unroll
      for (int rh = 0; rh < 2; ++rh)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          hw[rh][k] = 0u;                             // zero output past sequence_length (and for padding rows)
          if (active[rh]) {
            float hv[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int f = 4 * k + 2 * rh + e;
              const float zi = d[f] + (e ? ptx::bf16_hi(xw[rh][0][k]) : ptx::bf16_lo(xw[rh][0][k]));
              const float zj = d[16 + f] + (e ? ptx::bf16_hi(xw[rh][1][k]) : ptx::bf16_lo(xw[rh][1][k]));
              const float zf = d[32 + f] + (e ? ptx::bf16_hi(xw[rh][2][k]) : ptx::bf16_lo(xw[rh][2][k]));
              const float zo = d[48 + f] + (e ? ptx::bf16_hi(xw[rh][3][k]) : ptx::bf16_lo(xw[rh][3][k]));
              const float ai = ptx::fast_sigmoid(zi), aj = ptx::fast_tanh(zj), af = ptx::fast_sigmoid(zf), ao = ptx::fast_sigmoid(zo);
              const float c = af * cst[rh][k][e] + ai * aj;      // forget_bias (+1.0) is folded into the projected bias
              cst[rh][k][e] = c;
              hv[e] = ao * ptx::fast_tanh(c);
              d[f] = ai; d[16 + f] = aj; d[32 + f] = af; d[48 + f] = ao;
            }
            hw[rh][k] = ptx::pack_bf16x2(hv[0], hv[1]);
          }
        }
      if (w == 0) LSTM_TRACE_WG(wgi, 7);
      // ---- h_t slice first (it is on the critical path), bookkeeping stores afterwards
      if (s + 1 < p.T) {
        const int nb = (s + 1) & 1;
        uint8_t* my_slice = smem_a + nb * C::A_BYTES + wgi * C::HALF_A_BYTES + rank * C::SLICE_BYTES;
        uint8_t* hx_slice = hx_half + (size_t)nb * hx_buf_stride + rank * C::SLICE_BYTES;
        // a warp's 4-byte stores cover 8 rows x 16 B of one K-chunk: conflict-free in shared memory
        uint8_t* dst = my_slice + word_off;
#pragma unroll
        for (int rh = 0; rh < 2; ++rh)
#pragma unroll
          for (int k = 0; k < 4; ++k) *reinterpret_cast<uint32_t*>(dst + k * 1024 + rh * 128) = hw[rh][k];
        ptx::fence_proxy_async_smem();                      // generic-proxy smem writes -> async proxy (bulk copies, wgmma)
        if (w == 0) LSTM_TRACE_WG(wgi, 8);
        if (wgi == 0) ptx::bar_sync(1, 128);                // the half's slice is complete (named barrier 1 / 2 per half)
        else ptx::bar_sync(2, 128);
        if (w == 0) {
          if (lane == 0) {
            ptx::bulk_store_1d(hx_slice, my_slice, C::SLICE_BYTES);          // async proxy: smem -> global (L2)
            ptx::bulk_commit();
            asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");       // writes performed, not just the smem reads
            ptx::bulk_load_1d_mc(my_slice, hx_slice, C::SLICE_BYTES, &my_full[nb], (uint16_t)(((1u << CS) - 1) & ~(1u << rank)));
            ptx::mbar_arrive(&my_full[nb]);                                 // the local slice is already in place
          }
          __syncwarp();
          LSTM_TRACE_WG(wgi, 9);
        }
      }
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        if (okn[rh]) {
          __nv_bfloat16* lo = p.lstm_out + ((size_t)n[rh] * p.H + t[rh]) * 512 + dir * 256 + rank * UPC + 2 * q4;
#pragma unroll
          for (int k = 0; k < 4; ++k) *reinterpret_cast<uint32_t*>(lo + 8 * k) = hw[rh][k];
        }
        if (active[rh] && p.gates != nullptr) {
          // coalesced saved-state layout (common.cuh): a warp's stores of one (gate, K-chunk) cover 8 rows x 16 B = 128 B contiguous
          const size_t dts = (size_t)unit * p.T + s;
          const int row = wgi * C::HALF_ROWS + rr0 + 8 * rh;
          __nv_bfloat16* gs = p.gates + lstm_gate_off(dts, 0, rank * UPC, row) + 2 * q4;
          float* cs = p.csave + lstm_c_off(dts, rank * UPC, row) + 2 * (q4 & 1);
#pragma unroll
          for (int g = 0; g < 4; ++g)
#pragma unroll
            for (int k = 0; k < 4; ++k)
              *reinterpret_cast<uint32_t*>(gs + g * LSTM_GATE_STRIDE + k * LSTM_GCHUNK_STRIDE) =
                  ptx::pack_bf16x2(d[16 * g + 4 * k + 2 * rh], d[16 * g + 4 * k + 2 * rh + 1]);
#pragma unroll
          for (int k = 0; k < 4; ++k)      // units 8k + 2*q4 .. = 4-unit chunk 2k + q4/2, position 2*(q4&1)
            *reinterpret_cast<float2*>(cs + (2 * k + (q4 >> 1)) * LSTM_CCHUNK_STRIDE) = make_float2(cst[rh][k][0], cst[rh][k][1]);
        }
      }
      if (w == 0) LSTM_TRACE_WG(wgi, 10);
    }
  }

  __syncthreads();
  cluster_arrive_release();          // no CTA leaves (and frees its smem / mbarriers) while a peer may still write into it
  cluster_wait_acquire();
}

}  // namespace lstm
