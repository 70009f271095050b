// conv1 weight/bias gradient on the tensor cores (pool1 + ReLU backward folded in).   lib/lstm/train.py:81-83 (tf.gradients)
//
//   dW1[r][s][co] = sum over pre-pool positions (h, w) of  data[h+r-1][w+s-1] * G[h][w][co]        db1[co] = sum G
//   G = the pooled gradient d_a1 routed to the arg-max position of its 2x2 window where a1 > 0, zero elsewhere.
//
// The SIMT kernel (backward_kernels.cu) spends 36 masked FMAs per pooled (position, channel); as a GEMM the
// layer is a 64 x 9 output with K = 8.4 M positions, i.e. nothing for the tensor pipe -- what costs is building the operands,
// so they are arranged for the cheapest build:
//
//   D[128 x 64] += A[128 x K] * B[64 x K]^T     (bf16 in, f32 accumulate in registers for the WHOLE kernel: one epilogue per CTA)
//     K index = (pooled position, window slot dy*2+dx): the unpooled gradient is never materialised, a pooled value g lands in
//               the slot its arg-max names and the other three slots of that K quad are zero
//     A rows  0..63  channels, pooled rows 0,1 of the stage ("set 0");  rows 64..127 the same channels for pooled rows 2,3 ("set 1")
//     B rows  0..31  set 0: [9 taps of the patch, bf16 high part | 1.0 | 0 x6 | 9 taps, bf16 remainder | 0 x7]; rows 32..63 set 1
//   so the diagonal blocks D[set][set] hold dW (high + remainder columns add up to the f32 product: G is bf16 already, the pixel
//   is split x = xh + xl exactly) and column 9 (the row of ones) holds db; the off-diagonal blocks are ignored.
//
// Both operands are written by threads in the no-swizzle K-major layout [K chunk of 8][row][16 B] (LBO = rows*16, SBO = 128), the
// layout conv1_tc.cuh uses.  One 16-B entry = one row x 8 consecutive K = 2 adjacent pooled positions x 4 window slots.
// Channel c of a set sits in row (c & 7) * 8 + (c >> 3): a builder thread owns 8 consecutive channels (one uint4 of the NHWC
// gradient) and its 8 entry stores then fall into 8 different bank groups across the quarter-warp.
//
// Roles (480 threads): warps 0..3 = the MMA warpgroup (accumulator rows 0..63 and 64..127 as two register sets) and the final
// epilogue (row quadrants), warps 4..11 gradient (A) builders, warps 12..14 patch (B) builders + input staging.  4-stage operand
// ring; a stage = 4 pooled rows x 16 pooled columns = 64 pooled positions = 256 K per set = 16 wgmma (K = 16) per row set.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace conv1wg {

constexpr int NUM_THREADS = 480;
constexpr int A_WARP0 = 4, B_WARP0 = 12;
constexpr int A_THREADS = 256, B_THREADS = 96;
constexpr int NST = 4;
constexpr int CHUNKS = 16;                          // K chunks of 8 per set and stage
constexpr int A_BYTES = CHUNKS * 128 * 16;          // 32 KB
constexpr int B_BYTES = CHUNKS * 64 * 16;           // 16 KB
constexpr int IN_ROWS = 10, IN_STRIDE = 36;         // staged input: image rows 2*ho0-1 .. 2*ho0+8, columns -1 .. 32 (+2 pad)
constexpr int IN_BYTES = IN_ROWS * IN_STRIDE * 4;
constexpr int OFF_B = NST * A_BYTES;
constexpr int OFF_IN = OFF_B + NST * B_BYTES;
constexpr int OFF_BAR = OFF_IN + 2 * IN_BYTES;
constexpr int SMEM_BYTES = OFF_BAR + 128 + 1024;

struct Params {
  const __nv_bfloat16* d_a1;   // [N, W/2, 16, 64] gradient of the pooled activation
  const __nv_bfloat16* a1;     // same shape, pooled activation (ReLU mask)
  const uint8_t* am1;          // same shape, window index dy*2+dx of the maximum
  const void* data;            // [N, W, 32] f32 or uint8 (the kernel's TIn)
  float* dW;                   // [9][64], accumulated with atomics
  float* db;                   // [64]
  int N, W, tiles_per_img;     // tiles_per_img = ceil((W/2) / 4)
};

// one channel of one pooled position: bf16 bits of the gradient (0 where the activation was clipped) -> the two words of its K quad
__device__ __forceinline__ void quad_words(uint32_t gbits, uint32_t idx, uint32_t& w01, uint32_t& w23) {
  const uint32_t v = (idx & 1u) ? (gbits << 16) : gbits;
  w01 = (idx & 2u) ? 0u : v;
  w23 = (idx & 2u) ? v : 0u;
}

// TIn: float (the f32 data tensor) or uint8_t (pixel bytes, widened to the same f32 values when they are staged: common.cuh)
template <typename TIn = float>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv1_wgrad_tc_kernel(const Params p) {
  using Px = Pixels4<TIn>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + OFF_B;
  float* s_in = reinterpret_cast<float*>(smem + OFF_IN);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + OFF_BAR);     // [NST]
  uint64_t* empty = full + NST;                                     // [NST]

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int H1 = p.W >> 1;
  const int num_tiles = p.N * p.tiles_per_img;

  if (warp_idx == 0 && lane == 0) {
    for (int s = 0; s < NST; ++s) {
      ptx::mbar_init(&full[s], A_THREADS + B_THREADS);
      ptx::mbar_init(&empty[s], 1);
    }
    ptx::fence_barrier_init();
  }
  // B: zero everything once, then the row of ones (tap slot 9 of the high part) of both sets; builders only ever write taps 0..8
  for (int e = threadIdx.x; e < NST * B_BYTES / 16; e += NUM_THREADS) {
    const int row = e & 63;
    const uint32_t one2 = ((row & 31) == 9) ? 0x3F803F80u : 0u;
    *reinterpret_cast<uint4*>(smem_b + (size_t)e * 16) = make_uint4(one2, one2, one2, one2);
  }
  ptx::fence_proxy_async_smem();
  __syncthreads();

  if (warp_idx < A_WARP0) {
    // ===================== MMA warpgroup, then the final epilogue: row = (set, row of the set), columns set*32 .. = [taps hi | ones | taps lo]
    float d0[32], d1[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { d0[i] = 0.f; d1[i] = 0.f; }
    int st = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      ptx::mbar_wait(&full[st], ph);
      const uint32_t a_base = ptx::smem_u32(smem_a + st * A_BYTES), b_base = ptx::smem_u32(smem_b + st * B_BYTES);
      wg::fence();
#pragma unroll
      for (int k = 0; k < CHUNKS / 2; ++k) {
        const uint64_t bd = ptx::make_desc_k_nosw(b_base + k * 2 * 1024, 1024, 128);
        wg::mma_bf16<64>(d0, ptx::make_desc_k_nosw(a_base + k * 2 * 2048, 2048, 128), bd, 1u);
        wg::mma_bf16<64>(d1, ptx::make_desc_k_nosw(a_base + 64 * 16 + k * 2 * 2048, 2048, 128), bd, 1u);
      }
      wg::commit();
      wg::wait<0>();
      if (threadIdx.x == 0) ptx::mbar_arrive(&empty[st]);
      if (++st == NST) { st = 0; ph ^= 1; }
    }
    wg::fence_operand(d0);
    wg::fence_operand(d1);
    // every builder write has been consumed: the A ring is free and holds the staged accumulators [128][64] f32
    float* acc_tile = reinterpret_cast<float*>(smem_a);
    ptx::acc_store<64, 64>(acc_tile, d0, 0);
    ptx::acc_store<64, 64>(acc_tile, d1, 64);
    ptx::bar_sync(1, 128);
    const int q = warp_idx & 3;
    const int set = q >> 1;
    const int mm = (q & 1) * 32 + lane;                      // row within the set
    const int ch = (mm & 7) * 8 + (mm >> 3);
    uint32_t v[32];
    ptx::acc_ld<64, 32>(acc_tile, q * 32 + lane, set * 32, v);
    if ((int)blockIdx.x < num_tiles) {
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) atomicAdd(p.dW + tap * 64 + ch, __uint_as_float(v[tap]) + __uint_as_float(v[16 + tap]));
      atomicAdd(p.db + ch, __uint_as_float(v[9]));
    }
  } else if (warp_idx >= B_WARP0) {
    // ===================== patch (B) builders + input staging =====================
    const int bt = threadIdx.x - B_WARP0 * 32;              // 0..95: item (chunk 0..15, set, kernel row r)
    const int r = bt % 3, cs = bt / 3;
    const int set = cs & 1, chunk = cs >> 1;
    const int hol = set * 2 + (chunk >> 3), pw = chunk & 7;  // pooled row within the stage, pair of pooled columns
    auto fetch = [&](int tile, typename Px::Raw& v) {
      const int n = tile / p.tiles_per_img;
      const int ho0 = (tile - n * p.tiles_per_img) * 4;
      const int rr = bt >> 3, c4 = bt & 7;
      const int gr = 2 * ho0 - 1 + rr;
      v = Px::zero();
      if (bt < IN_ROWS * 8 && gr >= 0 && gr < p.W) v = Px::load(static_cast<const TIn*>(p.data) + ((size_t)n * p.W + gr) * 32, c4);
    };
    auto stash = [&](float* stg, const typename Px::Raw& raw) {
      if (bt < IN_ROWS * 8) {
        const float4 v = Px::f32(raw);
        float* d = stg + (bt >> 3) * IN_STRIDE + 1 + (bt & 7) * 4;    // image column c lives at index c + 1
        d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
      }
    };
    for (int b = 0; b < 2; ++b)                               // zero halo columns (image columns -1 and 32) of both stages, once
      if (bt < IN_ROWS) {
        float* rowp = s_in + b * IN_ROWS * IN_STRIDE + bt * IN_STRIDE;
        rowp[0] = 0.f; rowp[33] = 0.f; rowp[34] = 0.f; rowp[35] = 0.f;
      }
    // input rows are prefetched TWO tiles ahead in registers (a tile is about one HBM round trip of work: one tile ahead
    // left the load latency exposed every iteration) and parked in the other s_in buffer one tile ahead
    const int G = gridDim.x;
    typename Px::Raw pre[2];
    if ((int)blockIdx.x < num_tiles) {
      fetch(blockIdx.x, pre[0]);
      stash(s_in, pre[0]);
    }
    if ((int)blockIdx.x + G < num_tiles) fetch(blockIdx.x + G, pre[1]);
    int st = 0, it = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles;) {
#pragma unroll
      for (int u = 0; u < 2; ++u) {                          // u == it & 1: pre[u] held tile `it` (already parked), pre[u ^ 1] holds tile it+1
        if (tile >= num_tiles) break;
        float* stg = s_in + u * (IN_ROWS * IN_STRIDE);
        if (tile + 2 * G < num_tiles) fetch(tile + 2 * G, pre[u]);
        asm volatile("bar.sync 3, %0;" ::"n"(B_THREADS) : "memory");     // this tile's input rows are parked (and the other buffer is free)
        ptx::mbar_wait(&empty[st], ph ^ 1);
        // rows 2*hol + r (+1) of the stage, columns 4*pw .. 4*pw+5 (index = image column + 1 -> the patch column origin)
        float R[2][6];
#pragma unroll
        for (int dy = 0; dy < 2; ++dy) {
          const float2* src = reinterpret_cast<const float2*>(stg + (2 * hol + r + dy) * IN_STRIDE + 4 * pw);
#pragma unroll
          for (int c = 0; c < 3; ++c) { const float2 t = src[c]; R[dy][2 * c] = t.x; R[dy][2 * c + 1] = t.y; }
        }
        uint8_t* sb = smem_b + st * B_BYTES + chunk * 1024 + set * 32 * 16;
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          // K order of the entry: [position 0: slots (0,0) (0,1) (1,0) (1,1) | position 1: the same], slot (dy,dx) reads R[dy][s + 2*pi + dx]
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int pi = 0; pi < 2; ++pi)
#pragma unroll
            for (int dy = 0; dy < 2; ++dy) {
              const float x0 = R[dy][s + 2 * pi], x1 = R[dy][s + 2 * pi + 1];
              const uint32_t h = ptx::pack_bf16x2(x0, x1);
              hi[pi * 2 + dy] = h;
              lo[pi * 2 + dy] = ptx::pack_bf16x2(x0 - ptx::bf16_lo(h), x1 - ptx::bf16_hi(h));
            }
          const int tap = r * 3 + s;
          *reinterpret_cast<uint4*>(sb + tap * 16) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
          *reinterpret_cast<uint4*>(sb + (16 + tap) * 16) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
        ptx::fence_proxy_async_smem();
        ptx::mbar_arrive(&full[st]);
        if (tile + G < num_tiles) stash(s_in + (u ^ 1) * (IN_ROWS * IN_STRIDE), pre[u ^ 1]);   // loaded a full tile ago
        tile += G; ++it;
        if (++st == NST) { st = 0; ph ^= 1; }
      }
    }
  } else if (warp_idx >= A_WARP0) {
    // ===================== gradient (A) builders =====================
    const int at = threadIdx.x - A_WARP0 * 32;              // 0..255: item (pair of pooled columns 0..31, channel group 0..7)
    const int cg = at & 7, pair = at >> 3;
    const int hol = pair >> 3, pw = pair & 7;
    const int set = hol >> 1, chunk = (hol & 1) * 8 + pw;
    const uint32_t a_off = chunk * 2048 + (set * 64 + cg) * 16;      // + j * 128 for channel j of the group
    auto fetch = [&](int tile, uint4 (&g)[2], uint4 (&y)[2], uint2 (&ix)[2]) {
      const int n = tile / p.tiles_per_img;
      const int ho = (tile - n * p.tiles_per_img) * 4 + hol;
#pragma unroll
      for (int pi = 0; pi < 2; ++pi) {
        if (ho < H1) {
          const size_t oo = (((size_t)n * H1 + ho) * 16 + 2 * pw + pi) * 64 + cg * 8;
          g[pi] = __ldg(reinterpret_cast<const uint4*>(p.d_a1 + oo));
          y[pi] = __ldg(reinterpret_cast<const uint4*>(p.a1 + oo));
          ix[pi] = __ldg(reinterpret_cast<const uint2*>(p.am1 + oo));
        } else {
          g[pi] = make_uint4(0u, 0u, 0u, 0u); y[pi] = g[pi]; ix[pi] = make_uint2(0u, 0u);
        }
      }
    };
    // three register slots, loads issued TWO tiles ahead (one tile is about one HBM round trip: see the patch builders)
    const int G = gridDim.x;
    uint4 g[3][2], y[3][2];
    uint2 ix[3][2];
    if ((int)blockIdx.x < num_tiles) fetch(blockIdx.x, g[0], y[0], ix[0]);
    if ((int)blockIdx.x + G < num_tiles) fetch(blockIdx.x + G, g[1], y[1], ix[1]);
    int st = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles;) {
#pragma unroll
      for (int u = 0; u < 3; ++u) {
        if (tile >= num_tiles) break;
        if (tile + 2 * G < num_tiles) fetch(tile + 2 * G, g[(u + 2) % 3], y[(u + 2) % 3], ix[(u + 2) % 3]);
        ptx::mbar_wait(&empty[st], ph ^ 1);
        uint8_t* sa = smem_a + st * A_BYTES + a_off;
        const uint32_t* gw0 = reinterpret_cast<const uint32_t*>(&g[u][0]);
        const uint32_t* gw1 = reinterpret_cast<const uint32_t*>(&g[u][1]);
        const uint32_t* yw0 = reinterpret_cast<const uint32_t*>(&y[u][0]);
        const uint32_t* yw1 = reinterpret_cast<const uint32_t*>(&y[u][1]);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int sh = (j & 1) * 16;
          // a1 is post-ReLU (>= 0): "a1 > 0" is "bf16 bits, sign aside, non-zero"
          const uint32_t y0 = (yw0[j >> 1] >> sh) & 0x7FFFu, y1 = (yw1[j >> 1] >> sh) & 0x7FFFu;
          const uint32_t g0 = y0 ? ((gw0[j >> 1] >> sh) & 0xFFFFu) : 0u, g1 = y1 ? ((gw1[j >> 1] >> sh) & 0xFFFFu) : 0u;
          const uint32_t i0 = ((j < 4 ? ix[u][0].x : ix[u][0].y) >> ((j & 3) * 8)) & 3u;
          const uint32_t i1 = ((j < 4 ? ix[u][1].x : ix[u][1].y) >> ((j & 3) * 8)) & 3u;
          uint4 e;
          quad_words(g0, i0, e.x, e.y);
          quad_words(g1, i1, e.z, e.w);
          *reinterpret_cast<uint4*>(sa + j * 128) = e;
        }
        ptx::fence_proxy_async_smem();
        ptx::mbar_arrive(&full[st]);
        tile += G;
        if (++st == NST) { st = 0; ph ^= 1; }
      }
    }
  }
}

}  // namespace conv1wg

// `u8`: `data` holds uint8 pixels (crnn_backward_u8), else f32
static int launch_conv1_wgrad_tc(const __nv_bfloat16* d_a1, const __nv_bfloat16* a1, const uint8_t* am1, const void* data, bool u8, float* dW,
                                 float* db, int N, int W, int num_sms, cudaStream_t st) {
  conv1wg::Params p;
  p.d_a1 = d_a1; p.a1 = a1; p.am1 = am1; p.data = data; p.dW = dW; p.db = db; p.N = N; p.W = W;
  p.tiles_per_img = ((W >> 1) + 3) / 4;
  static bool attr = false;
  if (!attr) {
    CUDA_TRY(cudaFuncSetAttribute(conv1wg::conv1_wgrad_tc_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, conv1wg::SMEM_BYTES));
    CUDA_TRY(cudaFuncSetAttribute(conv1wg::conv1_wgrad_tc_kernel<uint8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, conv1wg::SMEM_BYTES));
    attr = true;
  }
  const int tiles = N * p.tiles_per_img;
  const int grid = tiles < num_sms ? tiles : num_sms;
  if (u8) conv1wg::conv1_wgrad_tc_kernel<uint8_t><<<grid, conv1wg::NUM_THREADS, conv1wg::SMEM_BYTES, st>>>(p);
  else conv1wg::conv1_wgrad_tc_kernel<float><<<grid, conv1wg::NUM_THREADS, conv1wg::SMEM_BYTES, st>>>(p);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
