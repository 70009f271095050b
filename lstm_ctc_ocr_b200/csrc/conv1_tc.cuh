// conv1 (3x3 SAME, 1 -> 64, bias, ReLU) + pool1 (2x2/2) on the tensor cores.   lib/networks/LSTM_train.py:24-25
//
// The SIMT kernel (kernels.cu) sits on the FP32 FMA ceiling of the chip (288 FMAs per pooled output vector; FFMA2 packs
// them into 144 instructions but not into fewer pipe cycles).  As a GEMM the layer is tiny
// (K = 9) -- what costs is moving 8.4 M positions x 64 channels through an epilogue -- so the operands are arranged for the
// cheapest epilogue:
//
//   D[128 x 256] = A[128 x 64] * B[256 x 64]^T        (bf16 in, f32 accumulate, four K = 16 wgmma per warpgroup and tile)
//     A = [ W' 0 ; 0 W' ] rows 0..63  : the 64 filters against K columns 0..31
//                         rows 64..127: the same filters against K columns 32..63
//     B row j             K 0..31  = the 3x3 patch of position j of image rows h0..h0+7   (j = hl*32 + w)
//                         K 32..63 = the patch of the position 8 image rows further down
//   so one tile covers 16 image rows x 32 = 512 positions, accumulator LANE = (row set, channel) and COLUMN = position:
//   the 2x2 pool is register-local in the epilogue thread and a warp stores 32 consecutive channels (64 B).
//
// f32 fidelity on a bf16 pipe: pixels and taps are split x = xh + xl, w = wh + wl (bf16 high part + bf16 remainder) and the 32
// K columns of a patch hold  [xh (9) 0 | xl (9) 0 | xh (9) 0 | 0 0]  against  [wh 0 | wh 0 | wl 0 | 0 0]  (10 columns per part, so
// every bf16x2 word is one F2FP of two neighbouring taps):  xh*wh + xl*wh + xh*wl reproduces the
// f32 product to ~2^-17 (the dropped xl*wl term), so the layer keeps the numerics of the f32 SIMT kernel it replaces: what is
// left of the error is the bf16 rounding of the OUTPUT.
//
// Both operands are written by threads (im2col in shared memory, no TMA): no-swizzle K-major layout
// [K-chunk of 8][row][16 B] (8-row x 16-B core matrices; LBO = rows*16, SBO = 128).  Roles (384 threads): warps 0..3 im2col
// builders (double-buffered B tile and input stage, so the build of tile i+1 overlaps the MMA + epilogue of tile i), warps
// 4..11 = two MMA warpgroups (accumulator rows 0..63 / 64..127) and the epilogue (row quadrant x column half) reading the
// accumulators staged in shared memory.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace conv1tc {

constexpr int NUM_THREADS = 384;
constexpr int BUILD_WARP0 = 0, BUILD_THREADS = 128;
constexpr int KCH = 8;                           // K-chunks of 8 bf16: 4 per row set
constexpr int A_BYTES = KCH * 128 * 16;          // [8 K-chunks][128 rows][16 B]
constexpr int B_BYTES = KCH * 256 * 16;          // [8 K-chunks][256 rows][16 B]
constexpr int IN_ROWS = 18, IN_STRIDE = 36;      // staged input: image rows h0-1 .. h0+16, columns -1 .. 32 (+2 pad)
constexpr int IN_BYTES = IN_ROWS * IN_STRIDE * 4;
constexpr int OFF_B = A_BYTES;
constexpr int OFF_IN = OFF_B + 2 * B_BYTES;
constexpr int OFF_ACC = (OFF_IN + 2 * IN_BYTES + 15) / 16 * 16;   // staged accumulators [128][256] f32
constexpr int OFF_BAR = OFF_ACC + 128 * 256 * 4;
constexpr int SMEM_BYTES = OFF_BAR + 128 + 1024;

// K column k (0..31) of a patch: part = k / 10 (x: hi, lo, hi | w: hi, hi, lo), tap = k % 10; tap 9 and k >= 30 are zero padding
__device__ __forceinline__ uint32_t bf16_bits(float v) { return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(v)); }
__device__ __forceinline__ float bf16_back(uint32_t b) { return __uint_as_float(b << 16); }

struct Params {
  const float* data;        // [N, W, 32] f32
  const float* wgt;         // HWIO [3,3,1,64]
  const float* bias;        // [64]
  __nv_bfloat16* out;       // [N, W/2, 16, 64]
  uint8_t* argmax;          // TRAIN: window index (dy*2+dx) of the max, same shape as out
  int N, W, tiles_per_img;  // tiles_per_img = ceil(W / 16)
};

template <bool TRAIN>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv1_tc_kernel(const Params p) {
  extern __shared__ uint8_t smem_raw[];
  // aligned by OFFSET (not by casting through an integer): the pointers stay in the shared address space -> LDS/STS, not LD/ST
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + OFF_B;
  float* s_in = reinterpret_cast<float*>(smem + OFF_IN);
  uint64_t* b_full = reinterpret_cast<uint64_t*>(smem + OFF_BAR);   // [2]
  uint64_t* b_empty = b_full + 2;
  float* acc_tile = reinterpret_cast<float*>(smem + OFF_ACC);

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.N * p.tiles_per_img;

  if (warp_idx == 0 && lane == 0) {
    for (int s = 0; s < 2; ++s) {
      ptx::mbar_init(&b_full[s], BUILD_THREADS);
      ptx::mbar_init(&b_empty[s], 2);          // one arrive per MMA warpgroup
    }
    ptx::fence_barrier_init();
  }
  // A = [W' 0; 0 W']: entry (chunk, row) = 16 B = 8 bf16 of K
  for (int e = threadIdx.x; e < KCH * 128; e += NUM_THREADS) {
    const int chunk = e >> 7, row = e & 127;
    const int ch = row & 63, set = row >> 6;
    uint32_t hw[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) hw[i] = 0u;
    if ((chunk >> 2) == set) {
      for (int i = 0; i < 8; ++i) {
        const int k = (chunk & 3) * 8 + i;
        const int part = k / 10, tap = k - part * 10;
        if (part < 3 && tap < 9) {
          const float wv = __ldg(p.wgt + tap * 64 + ch);
          const uint32_t hi = bf16_bits(wv);
          hw[i] = (part == 2) ? bf16_bits(wv - bf16_back(hi)) : hi;
        }
      }
    }
    *reinterpret_cast<uint4*>(smem_a + chunk * 2048 + row * 16) =
        make_uint4(hw[0] | (hw[1] << 16), hw[2] | (hw[3] << 16), hw[4] | (hw[5] << 16), hw[6] | (hw[7] << 16));
  }
  ptx::fence_proxy_async_smem();
  __syncthreads();

  if (warp_idx < BUILD_WARP0 + 4) {
    // ===================== im2col builders =====================
    const int bt = threadIdx.x - BUILD_WARP0 * 32;          // 0..127
    // staged input of a tile: image rows h0-1 .. h0+16 (zero outside the image) = 144 float4; thread bt owns entries bt and
    // bt+128.  The loads of tile i+1 are issued BEFORE tile i is built and land in shared memory after it, so their
    // L2/HBM latency is off the per-tile critical path (a tile is a short piece of builder work).
    auto fetch = [&](int tile, float4 (&v)[2]) {
      const int n = tile / p.tiles_per_img;
      const int h0 = (tile - n * p.tiles_per_img) * 16;
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int e = bt + k * BUILD_THREADS;
        const int r = e >> 3, c4 = e & 7;
        const int gr = h0 - 1 + r;
        v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (e < IN_ROWS * 8 && gr >= 0 && gr < p.W) v[k] = __ldg(reinterpret_cast<const float4*>(p.data + ((size_t)n * p.W + gr) * 32) + c4);
      }
    };
    auto stash = [&](float* stg, const float4 (&v)[2]) {
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int e = bt + k * BUILD_THREADS;
        if (e < IN_ROWS * 8) {
          float* d = stg + (e >> 3) * IN_STRIDE + 1 + (e & 7) * 4;
          d[0] = v[k].x; d[1] = v[k].y; d[2] = v[k].z; d[3] = v[k].w;
        }
      }
    };
    for (int b = 0; b < 2; ++b)                               // zero halo columns of both stages, once
      if (bt < IN_ROWS) { s_in[b * IN_ROWS * IN_STRIDE + bt * IN_STRIDE] = 0.f; s_in[b * IN_ROWS * IN_STRIDE + bt * IN_STRIDE + 33] = 0.f; }
    float4 pre[2];
    if (blockIdx.x < num_tiles) {
      fetch(blockIdx.x, pre);
      stash(s_in, pre);
    }
    int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int st = it & 1;
      const uint32_t ph = (it >> 1) & 1;
      float* stg = s_in + st * (IN_ROWS * IN_STRIDE);
      const int nxt = tile + gridDim.x;
      if (nxt < num_tiles) fetch(nxt, pre);
      asm volatile("bar.sync 2, %0;" ::"n"(BUILD_THREADS) : "memory");
      ptx::mbar_wait(&b_empty[st], ph ^ 1);                  // the MMAs that read this B buffer two tiles ago have retired
      uint8_t* sb = smem_b + st * B_BYTES;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int j = bt + rr * BUILD_THREADS;               // B row: position (hl, w) of both row sets
        const int hl = j >> 5, w = j & 31;
#pragma unroll
        for (int set = 0; set < 2; ++set) {
          const float* s0 = stg + (hl + set * 8) * IN_STRIDE + w;   // patch origin: image row h-1, column w-1
          float x[10];
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int s = 0; s < 3; ++s) x[r * 3 + s] = s0[r * IN_STRIDE + s];
          x[9] = 0.f;
          uint32_t wd[16];                                    // K pairs: [hi x5 | lo x5 | hi x5 | 0]
#pragma unroll
          for (int m = 0; m < 5; ++m) {
            const uint32_t h = ptx::pack_bf16x2(x[2 * m], x[2 * m + 1]);                         // one F2FP per two taps
            wd[m] = h; wd[10 + m] = h;
            wd[5 + m] = ptx::pack_bf16x2(x[2 * m] - ptx::bf16_lo(h), x[2 * m + 1] - ptx::bf16_hi(h));
          }
          wd[15] = 0u;
#pragma unroll
          for (int cq = 0; cq < 4; ++cq)
            *reinterpret_cast<uint4*>(sb + (set * 4 + cq) * 4096 + j * 16) = make_uint4(wd[4 * cq], wd[4 * cq + 1], wd[4 * cq + 2], wd[4 * cq + 3]);
        }
      }
      ptx::fence_proxy_async_smem();
      ptx::mbar_arrive(&b_full[st]);
      if (nxt < num_tiles) stash(s_in + (st ^ 1) * (IN_ROWS * IN_STRIDE), pre);
    }
  } else {
    // ===================== MMA (rows wgi*64 ..) + epilogue: row = (row set, channel), columns = positions =====================
    const int wgi = (warp_idx >> 2) - 1;
    const bool arriver = (warp_idx & 3) == 0 && lane == 0;
    const int q = warp_idx & 3;
    const int half = (warp_idx - 4) >> 2;                    // columns half*128 ..: image rows half*4 .. half*4+3 of the set
    const int set = q >> 1;
    const int c = (q & 1) * 32 + lane;
    const float bias = __ldg(p.bias + c), nbias = -bias;
    const int Hp = p.W >> 1;
    int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int st = it & 1;
      const int n = tile / p.tiles_per_img;
      const int h0 = (tile - n * p.tiles_per_img) * 16;
      ptx::mbar_wait(&b_full[st], (it >> 1) & 1);
      {
        float d[128];
        const uint32_t a_base = ptx::smem_u32(smem_a) + wgi * 64 * 16, b_base = ptx::smem_u32(smem_b + st * B_BYTES);
        wg::fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wg::mma_bf16<256>(d, ptx::make_desc_k_nosw(a_base + k * 2 * 2048, 2048, 128), ptx::make_desc_k_nosw(b_base + k * 2 * 4096, 4096, 128),
                            k != 0);
        wg::commit();
        wg::wait<0>();
        wg::fence_operand(d);
        if (arriver) ptx::mbar_arrive(&b_empty[st]);
        ptx::bar_sync(1, 256);                               // the previous tile's epilogue reads are done
        ptx::acc_store<256, 256>(acc_tile, d, wgi * 64);
        ptx::bar_sync(1, 256);
      }
      const int c0 = half * 128, arow = q * 32 + lane;
#pragma unroll 1
      for (int pr = 0; pr < 2; ++pr) {
        uint32_t v0[32], v1[32];
        ptx::acc_ld<256, 32>(acc_tile, arow, c0 + pr * 64, v0);        // image row h   (32 columns)
        ptx::acc_ld<256, 32>(acc_tile, arow, c0 + pr * 64 + 32, v1);   // image row h+1
        const int h = h0 + set * 8 + half * 4 + 2 * pr;
        if (h < p.W) {                                        // W is even: both rows of a window are inside or outside together
          const size_t off = (((size_t)n * Hp + (h >> 1)) * 16) * 64 + c;
#pragma unroll
          for (int pw = 0; pw < 16; ++pw) {
            const float x00 = __uint_as_float(v0[2 * pw]), x01 = __uint_as_float(v0[2 * pw + 1]);
            const float x10 = __uint_as_float(v1[2 * pw]), x11 = __uint_as_float(v1[2 * pw + 1]);
            if (!TRAIN) {
              // relu(max4 + b) == max(max4, -b) + b exactly (the same FADD on the same operand, or (-b) + b = 0): two 3-input
              // maxima and one add instead of three maxima, an add and a max -- the epilogue is ALU-issue bound
              const float m4 = fmaxf(fmaxf(fmaxf(x00, x01), fmaxf(x10, x11)), nbias);
              const float o = m4 + bias;
              reinterpret_cast<unsigned short*>(p.out)[off + (size_t)pw * 64] = (unsigned short)ptx::pack_bf16x2(o, o);   // F2FP (ALU), not F2F (XU)
            } else {
              // strict '>' in (dy, dx) row-major order keeps the FIRST maximum (tie-break of TF/torch max-pool gradients),
              // decided on the f32 accumulators like the SIMT kernel
              float best = x00;
              uint32_t bi = 0;
              if (x01 > best) { best = x01; bi = 1; }
              if (x10 > best) { best = x10; bi = 2; }
              if (x11 > best) { best = x11; bi = 3; }
              const float o = fmaxf(best + bias, 0.f);
              reinterpret_cast<unsigned short*>(p.out)[off + (size_t)pw * 64] = (unsigned short)ptx::pack_bf16x2(o, o);
              p.argmax[off + (size_t)pw * 64] = (uint8_t)bi;
            }
          }
        }
      }
    }
  }
}

}  // namespace conv1tc

static int launch_conv1_tc(const float* data, const float* w, const float* b, __nv_bfloat16* out, uint8_t* argmax, int N, int W,
                           int num_sms, cudaStream_t st) {
  conv1tc::Params p;
  p.data = data; p.wgt = w; p.bias = b; p.out = out; p.argmax = argmax; p.N = N; p.W = W; p.tiles_per_img = (W + 15) / 16;
  static bool attr = false;
  if (!attr) {
    CUDA_TRY(cudaFuncSetAttribute(conv1tc::conv1_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, conv1tc::SMEM_BYTES));
    CUDA_TRY(cudaFuncSetAttribute(conv1tc::conv1_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, conv1tc::SMEM_BYTES));
    attr = true;
  }
  const int tiles = N * p.tiles_per_img;
  const int grid = tiles < num_sms ? tiles : num_sms;
  if (argmax != nullptr) conv1tc::conv1_tc_kernel<true><<<grid, conv1tc::NUM_THREADS, conv1tc::SMEM_BYTES, st>>>(p);
  else conv1tc::conv1_tc_kernel<false><<<grid, conv1tc::NUM_THREADS, conv1tc::SMEM_BYTES, st>>>(p);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
