// Persistent backward recurrence (BPTT) of the BiLSTM for sm_90a; mirror image of csrc/lstm.cuh.
//
// Restates what tf.gradients produces for tf.contrib.rnn.LSTMCell under bidirectional_dynamic_rnn
// (lib/networks/network.py:104-107, lib/lstm/train.py:82).  Per step s = T-1 .. 0 (step space: frame t = s for the
// forward direction, len-1-s for the backward direction; inactive when s >= len):
//   dh = d_out[t] + dz_{s+1} W_h^T          dc = dc_{s+1->s} + dh * o * (1 - tanh(c_s)^2)
//   do = dh * tanh(c_s) * o(1-o)   di = dc * j * i(1-i)   dj = dc * i * (1-j^2)   df = dc * c_{s-1} * f(1-f)
//   dc_{s->s-1} = dc * f
// Cluster of 8 CTAs per (direction, 128-sample tile); CTA `rank` owns 32 hidden units and keeps dc for them in registers.
// The recurrent product is split along K and NOTHING but generic-proxy traffic passes between CTAs (details above the kernel).
// Outputs: dz for every (sample, frame) in FRAME order (`dz_all`, consumed by the dW_x / dW_h / dx GEMMs).
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "lstm.cuh"
#include "wgmma.cuh"

namespace lstm_bwd {

constexpr int BLOCK_M = 128;
constexpr int CS = 8;
constexpr int UPC = 32;

struct Params {
  const __nv_bfloat16* gates;     // saved by the forward kernel, coalesced per batch tile (common.cuh: lstm_gate_off)
  const float* csave;             // (common.cuh: lstm_c_off)
  const __nv_bfloat16* d_out;     // [Nimg*H, 512] gradient w.r.t. the LSTM output (frame order)
  __nv_bfloat16* dz_all;          // [Nimg*H, 2048] frame order, permuted gate columns, [fw | bw]
  const int* seq_len;
  int Nimg, Npad, H, T, tiles_per_dir;
};

__device__ __forceinline__ uint4 pack8(const float* v) {
  return make_uint4(ptx::pack_bf16x2(v[0], v[1]), ptx::pack_bf16x2(v[2], v[3]), ptx::pack_bf16x2(v[4], v[5]),
                    ptx::pack_bf16x2(v[6], v[7]));
}
__device__ __forceinline__ void unpack8(const uint4 q, float* v) {
  v[0] = ptx::bf16_lo(q.x); v[1] = ptx::bf16_hi(q.x); v[2] = ptx::bf16_lo(q.y); v[3] = ptx::bf16_hi(q.y);
  v[4] = ptx::bf16_lo(q.z); v[5] = ptx::bf16_hi(q.z); v[6] = ptx::bf16_lo(q.w); v[7] = ptx::bf16_hi(q.w);
}

// ---------------------------------------------------------------------------------------------------------------------------
// The recurrence with the product split along K ("ks").  Moving the whole dz_{s+1} tile (128 x 1024, 256 KB) into every CTA
// each step would mean MMAs of N = 32, a multicast ring with cluster-wide slot hand-shakes, two fence.proxy.async and a
// cluster barrier per step.  Instead CTA `rank` multiplies ONLY ITS OWN dz slice
// (128 x 128 gate columns, written by its own epilogue straight into shared memory as the no-swizzle A operand) with the
// resident W_h[all 256 units, its 128 gate columns]: 8 wgmma of 64 x 256 x 16 per warpgroup give its partial dh for ALL units.  The
// partials are exchanged all-to-all through L2 as bf16 (8 KB per (source, destination) pair): plain st.global, one
// release.cluster arrive on every peer's mbarrier, acquire.cluster wait, ld.global.cg of the 8 partial rows, f32 sum --
// no async proxy, no proxy fences, no cluster barrier on the critical path.
//   X[buf = s & 1][unit][dst][src][128 rows][32 units] bf16 is the exchange buffer (double buffered: a source can only reach
//   step s-2 after every peer finished reading step s, because its own step s-1 needs all peers' step s-1 partials).
namespace ks {
constexpr int NUM_THREADS = 384;                 // warpgroup 0 setup, warpgroups 1..2 MMA (rows 0..63 / 64..127) + epilogue
constexpr int EPI_THREADS = 256;
constexpr int B_BYTES = 2 * 256 * 128;           // 2 K-blocks x [256 unit rows x 128 B] (SW128) = 64 KB
constexpr int A_BYTES = 16 * BLOCK_M * 16;       // [16 K-chunks][128 rows][16 B] = 32 KB, no swizzle
constexpr int ACC_OFFSET = B_BYTES + A_BYTES;    // staged accumulators [128 rows][256] f32
constexpr int BAR_OFFSET = ACC_OFFSET + BLOCK_M * 256 * 4;
constexpr int SMEM_BYTES = BAR_OFFSET + 128 + 1024;
constexpr int PAIR_BYTES = BLOCK_M * UPC * 2;    // one (source, destination) block of partial sums: 8 KB
}  // namespace ks

__global__ void __launch_bounds__(ks::NUM_THREADS, 1)
lstm_bwd_ks_kernel(const __grid_constant__ CUtensorMap tmW, const Params p, uint8_t* __restrict__ xbuf) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_b = smem;
  uint8_t* smem_a = smem + ks::B_BYTES;
  float* acc_tile = reinterpret_cast<float*>(smem + ks::ACC_OFFSET);
  uint64_t* b_full = reinterpret_cast<uint64_t*>(smem + ks::BAR_OFFSET);
  uint64_t* a_ready = b_full + 1;
  uint64_t* part_ready = a_ready + 1;            // [2]

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = (int)lstm::cluster_ctarank();
  const int unit = blockIdx.x / CS;
  const int dir = unit / p.tiles_per_dir;
  const int tile = unit - dir * p.tiles_per_dir;
  const int num_units = 2 * p.tiles_per_dir;

  if (warp_idx == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmW);
    ptx::mbar_init(b_full, 1);
    ptx::mbar_init(a_ready, ks::EPI_THREADS);
    ptx::mbar_init(&part_ready[0], CS);
    ptx::mbar_init(&part_ready[1], CS);
    ptx::fence_barrier_init();
    // resident W_h[dir: all 256 units][gate columns rank*128 .. +128)
    ptx::mbar_arrive_expect_tx(b_full, ks::B_BYTES);
    for (int kb = 0; kb < 2; ++kb) ptx::tma_load_2d(&tmW, b_full, smem_b + kb * 256 * 128, rank * 128 + kb * 64, dir * 256);
  }
  __syncthreads();
  lstm::cluster_arrive_release();                  // peers arrive on this CTA's part_ready barriers
  lstm::cluster_wait_acquire();

  if (warp_idx < 4) {
    ptx::setmaxnreg_dec<40>();
  } else {
    // ===================== MMA: partial dh[128 x 256] = dz_{s+1}[128 x own 128 gate columns] * W_h^T; epilogue: thread = (sample row, half)
    ptx::setmaxnreg_inc<232>();
    const int wgi = (warp_idx >> 2) - 1;           // MMA rows wgi*64 ..
    const int q = warp_idx & 3;
    const int hh = (warp_idx - 4) >> 2;            // exchange: destination CTAs hh*4 .. hh*4+3; cell: units hh*16 .. +16 of this CTA
    const int u0 = hh * 16;
    const int row = q * 32 + lane;
    const int n = tile * BLOCK_M + row;
    const bool okn = n < p.Nimg;
    const int len = okn ? min(max(__ldg(p.seq_len + n), 0), p.T) : 0;
    ptx::mbar_wait(b_full, 0);
    float dcr[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) dcr[i] = 0.f;
    const size_t buf_stride = (size_t)num_units * CS * CS * ks::PAIR_BYTES;
    uint8_t* x_unit = xbuf + (size_t)unit * CS * CS * ks::PAIR_BYTES;

    for (int s = p.T - 1; s >= 0; --s) {
      const bool has_rec = (s < p.T - 1);
      const bool active = s < len;
      const int t = active ? (dir ? (len - 1 - s) : s) : s;
      const size_t dts = (size_t)unit * p.T + s;                    // coalesced saved-state layout, common.cuh
      // pull the next step's saved state into L2 one step ahead (it was evicted long ago)
      if (s >= 1 && (s - 1) < len) {
        const int tp = dir ? (len - s) : (s - 1);
#pragma unroll
        for (int g = 0; g < 4; ++g) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.gates + lstm_gate_off(dts - 1, g, rank * UPC + u0, row)));
        asm volatile("prefetch.global.L2 [%0];" ::"l"(p.csave + lstm_c_off(dts - 1, rank * UPC + u0, row)));
        if (s >= 2) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.csave + lstm_c_off(dts - 2, rank * UPC + u0, row)));
        asm volatile("prefetch.global.L2 [%0];" ::"l"(p.d_out + ((size_t)n * p.H + tp) * 512 + dir * 256 + rank * UPC + u0));
      }

      float rec[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) rec[i] = 0.f;
      if (has_rec) {
        const int b = s & 1;
        uint8_t* xb = x_unit + (size_t)b * buf_stride;
        ptx::mbar_wait(a_ready, (uint32_t)(p.T - 2 - s) & 1u);
        {
          float d[128];
          const uint32_t a_base = ptx::smem_u32(smem_a) + wgi * 64 * 16;
          wg::fence();
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const uint64_t a_desc = ptx::make_desc_k_nosw(a_base + k * 4096, 2048, 128);
            const uint64_t b_desc = ptx::make_desc_k_sw128(ptx::smem_u32(smem_b + (k >> 2) * 256 * 128)) + 2 * (k & 3);
            wg::mma_bf16<256>(d, a_desc, b_desc, k != 0);
          }
          wg::commit();
          wg::wait<0>();
          wg::fence_operand(d);
          ptx::acc_store<256, 256>(acc_tile, d, wgi * 64);
        }
        ptx::bar_sync(1, ks::EPI_THREADS);
        // ---- this CTA's partial sums for destinations hh*4 .. hh*4+3 -> X[dst][src = rank][row]
#pragma unroll 1
        for (int jj = 0; jj < 4; ++jj) {
          uint32_t v[32];
          ptx::acc_ld<256, 32>(acc_tile, row, hh * 128 + jj * 32, v);
          uint32_t w[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) w[i] = ptx::pack_bf16x2(__uint_as_float(v[2 * i]), __uint_as_float(v[2 * i + 1]));
          uint8_t* dst = xb + ((size_t)((hh * 4 + jj) * CS + rank) * BLOCK_M + row) * 64;
          ptx::st_global_v8(dst, w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7]);
          ptx::st_global_v8(dst + 32, w[8], w[9], w[10], w[11], w[12], w[13], w[14], w[15]);
        }
        asm volatile("bar.sync 1, %0;" ::"n"(ks::EPI_THREADS) : "memory");
        // one release.cluster arrive per peer (cumulative over the barrier above: covers every thread's stores)
        if (warp_idx == 4 && lane < CS) ptx::mbar_arrive_cluster(ptx::mapa(ptx::smem_u32(&part_ready[b]), (uint32_t)lane));
      }
      // saved forward state of this step: issued before the exchange wait so that its latency hides behind it
      uint4 qg[4][2], qd[2];
      float4 qc[4], qp[4];
      if (active) {
        const __nv_bfloat16* gs = p.gates + lstm_gate_off(dts, 0, rank * UPC + u0, row);
        const float* cs = p.csave + lstm_c_off(dts, rank * UPC + u0, row);
        const __nv_bfloat16* dout = p.d_out + ((size_t)n * p.H + t) * 512 + dir * 256 + rank * UPC + u0;
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          qg[g][0] = __ldg(reinterpret_cast<const uint4*>(gs + g * LSTM_GATE_STRIDE));
          qg[g][1] = __ldg(reinterpret_cast<const uint4*>(gs + g * LSTM_GATE_STRIDE + LSTM_GCHUNK_STRIDE));
        }
        qd[0] = __ldg(reinterpret_cast<const uint4*>(dout));
        qd[1] = __ldg(reinterpret_cast<const uint4*>(dout) + 1);
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          qc[v] = __ldg(reinterpret_cast<const float4*>(cs + v * LSTM_CCHUNK_STRIDE));
          qp[v] = (s > 0) ? __ldg(reinterpret_cast<const float4*>(cs - LSTM_CSTEP_STRIDE + v * LSTM_CCHUNK_STRIDE)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      if (has_rec) {
        const int b = s & 1;
        uint8_t* xb = x_unit + (size_t)b * buf_stride;
        // ---- all 8 partial rows for this thread's 16 units
        ptx::mbar_wait_cluster(&part_ready[b], (uint32_t)((p.T - 2 - s) >> 1) & 1u);
        const uint8_t* src = xb + ((size_t)(rank * CS) * BLOCK_M + row) * 64 + hh * 32;
#pragma unroll
        for (int r = 0; r < CS; ++r) {
          const uint4 a = __ldcg(reinterpret_cast<const uint4*>(src + (size_t)r * BLOCK_M * 64));
          const uint4 c = __ldcg(reinterpret_cast<const uint4*>(src + (size_t)r * BLOCK_M * 64) + 1);
          float f[16];
          unpack8(a, f);
          unpack8(c, f + 8);
#pragma unroll
          for (int i = 0; i < 16; ++i) rec[i] += f[i];
        }
      }

      float dzi[16], dzj[16], dzf[16], dzo[16];
      if (active) {
        float gi[16], gj[16], gf[16], go[16], dh[16];
        unpack8(qg[0][0], gi); unpack8(qg[0][1], gi + 8);
        unpack8(qg[1][0], gj); unpack8(qg[1][1], gj + 8);
        unpack8(qg[2][0], gf); unpack8(qg[2][1], gf + 8);
        unpack8(qg[3][0], go); unpack8(qg[3][1], go + 8);
        unpack8(qd[0], dh); unpack8(qd[1], dh + 8);
        const float* cc = reinterpret_cast<const float*>(qc);
        const float* cp = reinterpret_cast<const float*>(qp);
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const float dht = dh[i] + rec[i];
          const float tc = ptx::fast_tanh(cc[i]);
          const float dc = dcr[i] + dht * go[i] * (1.f - tc * tc);
          dzo[i] = dht * tc * go[i] * (1.f - go[i]);
          dzi[i] = dc * gj[i] * gi[i] * (1.f - gi[i]);
          dzj[i] = dc * gi[i] * (1.f - gj[i] * gj[i]);
          dzf[i] = dc * cp[i] * gf[i] * (1.f - gf[i]);
          dcr[i] = dc * gf[i];
        }
      } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) { dzi[i] = 0.f; dzj[i] = 0.f; dzf[i] = 0.f; dzo[i] = 0.f; }
      }
      const uint4 zi0 = pack8(dzi), zi1 = pack8(dzi + 8), zj0 = pack8(dzj), zj1 = pack8(dzj + 8);
      const uint4 zf0 = pack8(dzf), zf1 = pack8(dzf + 8), zo0 = pack8(dzo), zo1 = pack8(dzo + 8);
      if (s > 0) {
        // A operand of the next step's product: K index = gate*32 + unit -> chunks gate*4 + hh*2 + {0, 1}
        uint8_t* a = smem_a + (size_t)(hh * 2) * 2048 + row * 16;
        *reinterpret_cast<uint4*>(a + 0 * 8192) = zi0; *reinterpret_cast<uint4*>(a + 0 * 8192 + 2048) = zi1;
        *reinterpret_cast<uint4*>(a + 1 * 8192) = zj0; *reinterpret_cast<uint4*>(a + 1 * 8192 + 2048) = zj1;
        *reinterpret_cast<uint4*>(a + 2 * 8192) = zf0; *reinterpret_cast<uint4*>(a + 2 * 8192 + 2048) = zf1;
        *reinterpret_cast<uint4*>(a + 3 * 8192) = zo0; *reinterpret_cast<uint4*>(a + 3 * 8192 + 2048) = zo1;
        ptx::fence_proxy_async_smem();
        ptx::mbar_arrive(a_ready);
      }
      if (okn) {
        __nv_bfloat16* za = p.dz_all + ((size_t)n * p.H + t) * 2048 + dir * 1024 + rank * 128 + u0;
        ptx::st_global_v8(za + 0 * 32, zi0.x, zi0.y, zi0.z, zi0.w, zi1.x, zi1.y, zi1.z, zi1.w);
        ptx::st_global_v8(za + 1 * 32, zj0.x, zj0.y, zj0.z, zj0.w, zj1.x, zj1.y, zj1.z, zj1.w);
        ptx::st_global_v8(za + 2 * 32, zf0.x, zf0.y, zf0.z, zf0.w, zf1.x, zf1.y, zf1.z, zf1.w);
        ptx::st_global_v8(za + 3 * 32, zo0.x, zo0.y, zo0.z, zo0.w, zo1.x, zo1.y, zo1.z, zo1.w);
      }
    }
  }

  __syncthreads();
  lstm::cluster_arrive_release();                  // no CTA leaves while a peer may still arrive on its barriers
  lstm::cluster_wait_acquire();
}

}  // namespace lstm_bwd
