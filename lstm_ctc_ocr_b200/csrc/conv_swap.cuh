// conv2 + bias + ReLU + 2x2 max-pool (lib/networks/LSTM_train.py:26-27) with the GEMM operands SWAPPED:
//
//   D^T[128 out-channels x 256 positions, f32] = W[128 x K] (bf16, K-major) * X[256 positions x K]^T (bf16, K-major)
//
// Why: with Cout = 128 the position-major kernel (gemm.cuh, M = 128 positions, N = 128 channels) moves 8 KB of operands
// through shared memory per 128x128x16 MMA and feeds the tensor pipe worse than the wide layers.  Putting the 128 channels on
// the M side lets N be 256 POSITIONS: 12 KB per 128x256x16 MMA -- the same smem bytes per flop as the Cout = 256 layers.
//
// A tile = 16 H-rows x Wd(16) of one image = 256 positions; per K-block (= one 3x3 tap, Cin = 64) the producer issues two
// 4-D TMA boxes of 128 positions at (r-1, s-1)-shifted coordinates (OOB zero fill = SAME padding, also past the image end)
// and one 2-D box of the weights.  Accumulator lane = output channel, column = position, so the 2x2 pool is register-local
// in the epilogue thread (columns hl*16+w: window = {2pw, 2pw+1} x {row, row+1}); a warp stores 32 consecutive channels.
//
// Inference (TRAIN = false): the pool window is local to the accumulator fragment (w pair = columns 2c, 2c+1; H pair = 16 columns
// apart), so pool, bias, ReLU and bf16 rounding happen in registers; the 16 KB pooled tile is written transposed into shared
// memory and leaves through two asynchronous TMA stores while the next tile's MMAs run.
// Training and the data-gradient kernel below drain the accumulators through shared memory one 64-column slice at a time
// (128 x 64 f32 = 32 KB, ptx::acc_store_slice), which leaves room for a 4-stage ring.  Slice j holds the 32-column chunks 2j and
// 2j+1; the two warps of a quadrant take one chunk each (chunk = one pooled row pair here, RC rows of H in the data-gradient kernel).
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace convsw {

constexpr int STAGES = 4;                   // what fits next to the 32 KB staged accumulator slice
constexpr int SLICE_N = 64;                 // accumulator columns staged at a time
constexpr int W_BYTES = 128 * 128;          // weights: 128 channels x 64 K (128 B rows, SW128)
constexpr int X_BYTES = 256 * 128;          // activations: 256 positions x 64 K
constexpr int STAGE_BYTES = W_BYTES + X_BYTES;
constexpr int ACC_OFFSET = STAGES * STAGE_BYTES;
constexpr int BAR_OFFSET = ACC_OFFSET + 128 * SLICE_N * 4;
constexpr int SMEM_BYTES = BAR_OFFSET + 256 + 1024;
static_assert(SMEM_BYTES <= 232448, "opt-in shared memory per block (227 KB)");
constexpr int NUM_THREADS = 384;            // warpgroup 0 producer, warpgroups 1..2 MMA (channels 0..63 / 64..127) + epilogue
constexpr int NUM_TAPS = 9;

struct Params {
  int Nimg, H;            // this launch covers images img0 .. img0+Nimg-1 of [*, H, 16, 64] NHWC (H = image width / 2) -> [*, H/2, 8, 128]
  int img0;
  int tiles_per_img;      // ceil(H / 16)
  const float* bias;      // [128]
  __nv_bfloat16* out;
  uint8_t* argmax;        // TRAIN: window index (dy*2+dx) of the max, same shape as out
  const int* line_w;      // LINES: [images] clamped line widths (input columns); pooled rows >= line_w / 4 are stored as zero
  const float* oscale;    // FP8: out is e4m3 [*, H/2, 8, 128] = e4m3(pooled value / *oscale) (a power of two)
};

template <bool TRAIN, bool LINES = false, bool FP8 = false>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv2_swap_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmO,
                  const Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;
  float* acc_tile = reinterpret_cast<float*>(smem + ACC_OFFSET);

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.Nimg * p.tiles_per_img;

  if (warp_idx == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmX);
    ptx::prefetch_tmap(&tmW);
    if (!TRAIN) ptx::prefetch_tmap(&tmO);
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);        // one arrive per MMA warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp_idx < 4) {
    ptx::setmaxnreg_dec<40>();
    // ===================== TMA producer: lanes 0/1 = the two activation boxes, lane 2 = the weight box =====================
    if (warp_idx == 0 && lane < 3) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int nl = tile / p.tiles_per_img, n = p.img0 + nl;
        const int h0 = (tile - nl * p.tiles_per_img) * 16;
        for (int tap = 0; tap < NUM_TAPS; ++tap) {
          const int r = tap / 3, sx = tap - 3 * r;
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* st = smem + stage * STAGE_BYTES;
          if (lane == 0) ptx::mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
          if (lane < 2) ptx::tma_load_4d(&tmX, &full_bar[stage], st + W_BYTES + lane * (X_BYTES / 2), 0, sx - 1, h0 + lane * 8 + r - 1, n);
          else ptx::tma_load_2d(&tmW, &full_bar[stage], st, tap * 64, 0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<232>();
    const int wgi = (warp_idx >> 2) - 1;             // accumulator rows (output channels) wgi*64 ..
    const bool arriver = (warp_idx & 3) == 0 && lane == 0;
    int stage = 0;
    uint32_t phase = 0;
    const int q = warp_idx & 3;
    const int ch = (warp_idx - 4) >> 2;               // 32-column chunk of each staged slice
    const int c = q * 32 + lane;                       // output channel of this thread
    const float bias = __ldg(p.bias + c);
    const int Hp = p.H >> 1;
    // inference epilogue (fragment side): this thread's accumulator rows are channels f0 and f0 + 8
    const int t = threadIdx.x & 127, l = t & 31;
    const int f0 = wgi * 64 + 16 * (t >> 5) + (l >> 2);
    const float bias0 = __ldg(p.bias + f0), bias8 = __ldg(p.bias + f0 + 8);
    const bool even = ((l >> 2) & 1) == 0;           // lanes l and l ^ 4 hold channels f0 and f0 ^ 1
    const bool issuer = !TRAIN && threadIdx.x == 128;
    uint8_t* stg = smem + ACC_OFFSET;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int nl = tile / p.tiles_per_img, n = p.img0 + nl;
      const int h0 = (tile - nl * p.tiles_per_img) * 16;
      float d[128];
      int prev = -1;
      for (int kb = 0; kb < NUM_TAPS; ++kb) {
        ptx::mbar_wait(&full_bar[stage], phase);
        const uint64_t a_desc = ptx::make_desc_k_sw128(ptx::smem_u32(smem + stage * STAGE_BYTES + wgi * 64 * 128));
        const uint64_t b_desc = ptx::make_desc_k_sw128(ptx::smem_u32(smem + stage * STAGE_BYTES + W_BYTES));
        wg::fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wg::mma_bf16<256>(d, a_desc + 2 * k, b_desc + 2 * k, (kb | k) != 0);
        wg::commit();
        wg::wait<1>();
        if (prev >= 0 && arriver) ptx::mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wg::wait<0>();
      wg::fence_operand(d);
      if (prev >= 0 && arriver) ptx::mbar_arrive(&empty_bar[prev]);
      if (!TRAIN) {
        // Pool, bias, ReLU and bf16 rounding in registers: fragment column 8j + 2(l%4) + {0,1} is a w pair of H row j/2 of the
        // tile, the H row below it is column group j + 2.  The pooled tile (8 pooled rows x 8 x 128 channels, 16 KB) goes through
        // shared memory as two [64 positions][64 channels] SWIZZLE_128B boxes and leaves with two TMA stores (rows >= H/2 dropped).
        if (issuer) ptx::bulk_wait_read_all();       // the previous tile's stores have read the buffer
        ptx::bar_sync(1, 256);
        const int ph_end = LINES ? (__ldg(p.line_w + n) >> 2) - (h0 >> 1) : 8;   // pooled rows of this tile inside the line
        if constexpr (FP8) {
          // e4m3 output: the pooled tile is one [64 positions][128 channels] box of bytes; each lane writes its two channels' bytes
          // (lanes l, l ^ 4, l ^ 8, .. hold neighbouring channels of one position: the bytes of a 4-byte word, no bank conflict)
          const float inv_os = 1.f / __ldg(p.oscale);
#pragma unroll
          for (int ph = 0; ph < 8; ++ph) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int j = 4 * ph + e;
              const float m0 = fmaxf(fmaxf(d[4 * j], d[4 * j + 1]), fmaxf(d[4 * j + 8], d[4 * j + 9]));
              const float m8 = fmaxf(fmaxf(d[4 * j + 2], d[4 * j + 3]), fmaxf(d[4 * j + 10], d[4 * j + 11]));
              uint32_t q = ptx::pack_e4m3x2(fmaxf(m0 + bias0, 0.f) * inv_os, fmaxf(m8 + bias8, 0.f) * inv_os);
              if (LINES && ph >= ph_end) q = 0u;
              const int row = ph * 8 + 4 * e + (l & 3);
              uint8_t* rb = stg + row * 128;
              rb[(((f0 >> 4) ^ (row & 7)) << 4) + (f0 & 15)] = (uint8_t)(q & 0xFFu);
              rb[((((f0 + 8) >> 4) ^ (row & 7)) << 4) + ((f0 + 8) & 15)] = (uint8_t)(q >> 8);
            }
          }
          ptx::fence_proxy_async_smem();
          ptx::bar_sync(1, 256);
          if (issuer) {
            ptx::tma_store_4d(&tmO, stg, 0, 0, h0 >> 1, n);
            ptx::bulk_commit();
          }
          continue;
        }
#pragma unroll
        for (int ph = 0; ph < 8; ++ph) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int j = 4 * ph + e;
            const float m0 = fmaxf(fmaxf(d[4 * j], d[4 * j + 1]), fmaxf(d[4 * j + 8], d[4 * j + 9]));
            const float m8 = fmaxf(fmaxf(d[4 * j + 2], d[4 * j + 3]), fmaxf(d[4 * j + 10], d[4 * j + 11]));
            const uint32_t b0 = __bfloat16_as_ushort(__float2bfloat16_rn(fmaxf(m0 + bias0, 0.f)));
            const uint32_t b8 = __bfloat16_as_ushort(__float2bfloat16_rn(fmaxf(m8 + bias8, 0.f)));
            // exchange with lane l ^ 4 so that each lane holds an adjacent channel pair: (f0, f0 + 1) or (f0 + 7, f0 + 8)
            const uint32_t r = __shfl_xor_sync(0xffffffffu, even ? b8 : b0, 4);
            uint32_t word = even ? (b0 | (r << 16)) : (r | (b8 << 16));
            if (LINES && ph >= ph_end) word = 0u;
            const int row = ph * 8 + 4 * e + (l & 3), ch = even ? f0 : f0 + 7;     // pooled position, first channel of the pair
            *reinterpret_cast<uint32_t*>(stg + (ch >> 6) * 8192 + row * 128 + ((((ch >> 3) & 7) ^ (row & 7)) << 4) + ((ch & 7) << 1)) = word;
          }
        }
        ptx::fence_proxy_async_smem();
        ptx::bar_sync(1, 256);
        if (issuer) {
          ptx::tma_store_4d(&tmO, stg, 0, 0, h0 >> 1, n);
          ptx::tma_store_4d(&tmO, stg + 8192, 64, 0, h0 >> 1, n);
          ptx::bulk_commit();
        }
        continue;
      }
#pragma unroll
      for (int j = 0; j < 256 / SLICE_N; ++j) {
        ptx::bar_sync(1, 256);                         // the previous slice's (tile's) epilogue reads are done
        ptx::acc_store_slice<256, SLICE_N>(acc_tile, d, wgi * 64, j);
        ptx::bar_sync(1, 256);
        uint32_t v[32];
        ptx::acc_ld<SLICE_N, 32>(acc_tile, q * 32 + lane, ch * 32, v);   // chunk 2j+ch, columns: [row h (16 w) | row h+1 (16 w)]
        const int h = h0 + 2 * (2 * j + ch);
        if (h < p.H) {                                  // H is even: both rows of the window are inside or outside together
          const size_t off = (((size_t)n * Hp + (h >> 1)) * 8) * 128 + c;
#pragma unroll
          for (int pw = 0; pw < 8; ++pw) {
            const float x00 = __uint_as_float(v[2 * pw]), x01 = __uint_as_float(v[2 * pw + 1]);
            const float x10 = __uint_as_float(v[16 + 2 * pw]), x11 = __uint_as_float(v[16 + 2 * pw + 1]);
            {
              // key = (bf16 bits of relu(x + b) << 2) | (3 - window index): the largest value wins, ties go to the FIRST
              // window position in (dy, dx) row-major order (the rule of gemm.cuh EPI_RELU_POOL12_T over a 2x2 window)
              const uint32_t p0 = ptx::pack_bf16x2(fmaxf(x00 + bias, 0.f), fmaxf(x01 + bias, 0.f));
              const uint32_t p1 = ptx::pack_bf16x2(fmaxf(x10 + bias, 0.f), fmaxf(x11 + bias, 0.f));
              const uint32_t k0 = ((p0 & 0xFFFFu) << 2) | 3u, k1 = ((p0 >> 16) << 2) | 2u;
              const uint32_t k2 = ((p1 & 0xFFFFu) << 2) | 1u, k3 = ((p1 >> 16) << 2) | 0u;
              const uint32_t k = max(max(k0, k1), max(k2, k3));
              reinterpret_cast<unsigned short*>(p.out)[off + (size_t)pw * 128] = (unsigned short)(k >> 2);
              p.argmax[off + (size_t)pw * 128] = (uint8_t)(3u - (k & 3u));
            }
          }
        }
      }
    }
    if (issuer) ptx::bulk_wait_all();                  // the CTA's shared memory must outlive its last stores
  }
}


// ---------------------------------------------------------------------------------------------------------------------------
// DATA gradients of the narrow layers (conv2: 64 input channels, conv3_1: 128) with the same operand swap.  conv2:  d_a1[p, ci] = sum over taps, co of d_pre2[p + tap', co] * W'[ci][(tap', co)]
// is a 3x3 SAME convolution of the [N, H, 16, 128] gradient with the flipped / transposed kernel (Bd_c2, backward_kernels.cu):
// only 64 output channels.  Position-major (gemm.cuh, BLOCK_N = 64) it would run the MMA at N = 64, a quarter of the N = 256
// rate.  Here the 64 channels sit on the M side (rows 64..127 of the weight box are out of bounds of the
// tensor map, i.e. zero-filled by TMA: half of the M = 128 MMA is padding) and N is 256 positions: half the padded work at the
// full rate.  K-blocks = 9 taps x 2 blocks of 64 gradient channels.  Epilogue: lane = input channel (quadrants 0 and 1 only),
// column = position; plain bf16 store (the ReLU / pool1 backward is folded into conv1's weight-gradient kernel).
// ---------------------------------------------------------------------------------------------------------------------------
// Templated on the geometry so that conv3_1's data gradient (Cin = 128: N = 128 position-major, half the MMA rate) takes the same
// route: WD = positions per H row (16 / 8), CB = 64-channel blocks of the incoming gradient (2 / 4), MVALID = output channels (64 / 128).
struct DgradParams {
  int Nimg, H;            // gradient [Nimg, H, WD, 64*CB] -> [Nimg, H, WD, MVALID]
  int tiles_per_img;      // ceil(H / (256 / WD))
  __nv_bfloat16* out;
};

template <int WD, int CB, int MVALID>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_dgrad_swap_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const DgradParams p) {
  constexpr int NUM_KB = 9 * CB;             // 9 taps x CB channel blocks
  constexpr int RT = 256 / WD;               // H rows per tile (two TMA boxes of RT/2 rows)
  constexpr int RC = 32 / WD;                // H rows per 32-column accumulator chunk
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;
  float* acc_tile = reinterpret_cast<float*>(smem + ACC_OFFSET);

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.Nimg * p.tiles_per_img;

  if (warp_idx == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmX);
    ptx::prefetch_tmap(&tmW);
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);        // one arrive per MMA warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp_idx < 4) {
    ptx::setmaxnreg_dec<40>();
    if (warp_idx == 0 && lane < 3) {                          // lanes 0/1: the two 128-position gradient boxes, lane 2: the weight box
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n = tile / p.tiles_per_img;
        const int h0 = (tile - n * p.tiles_per_img) * RT;
        for (int kb = 0; kb < NUM_KB; ++kb) {
          const int tap = kb / CB, cb = kb - tap * CB;
          const int r = tap / 3, sx = tap - 3 * r;
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* st = smem + stage * STAGE_BYTES;
          if (lane == 0) ptx::mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
          if (lane < 2) ptx::tma_load_4d(&tmX, &full_bar[stage], st + W_BYTES + lane * (X_BYTES / 2), cb * 64, sx - 1, h0 + lane * (RT / 2) + r - 1, n);
          else ptx::tma_load_2d(&tmW, &full_bar[stage], st, kb * 64, 0);       // MVALID = 64: rows 64..127 out of bounds -> zero fill
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<232>();
    const int wgi = (warp_idx >> 2) - 1;             // accumulator rows (output channels) wgi*64 ..
    const bool arriver = (warp_idx & 3) == 0 && lane == 0;
    int stage = 0;
    uint32_t phase = 0;
    const int q = warp_idx & 3;
    const int ch = (warp_idx - 4) >> 2;      // 32-column chunk of each staged slice
    const int c = q * 32 + lane;              // input channel of this thread (valid for c < MVALID)
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int n = tile / p.tiles_per_img;
      const int h0 = (tile - n * p.tiles_per_img) * RT;
      float d[128];
      int prev = -1;
      for (int kb = 0; kb < NUM_KB; ++kb) {
        ptx::mbar_wait(&full_bar[stage], phase);
        const uint64_t a_desc = ptx::make_desc_k_sw128(ptx::smem_u32(smem + stage * STAGE_BYTES + wgi * 64 * 128));
        const uint64_t b_desc = ptx::make_desc_k_sw128(ptx::smem_u32(smem + stage * STAGE_BYTES + W_BYTES));
        wg::fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wg::mma_bf16<256>(d, a_desc + 2 * k, b_desc + 2 * k, (kb | k) != 0);
        wg::commit();
        wg::wait<1>();
        if (prev >= 0 && arriver) ptx::mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wg::wait<0>();
      wg::fence_operand(d);
      if (prev >= 0 && arriver) ptx::mbar_arrive(&empty_bar[prev]);
#pragma unroll
      for (int j = 0; j < 256 / SLICE_N; ++j) {
        ptx::bar_sync(1, 256);                         // the previous slice's (tile's) epilogue reads are done
        ptx::acc_store_slice<256, SLICE_N>(acc_tile, d, wgi * 64, j);
        ptx::bar_sync(1, 256);
        if (q * 32 < MVALID) {
          uint32_t v[32];
          ptx::acc_ld<SLICE_N, 32>(acc_tile, q * 32 + lane, ch * 32, v);     // chunk 2j+ch, columns: RC consecutive H rows of WD positions each
#pragma unroll
          for (int hr = 0; hr < RC; ++hr) {
            const int h = h0 + (2 * j + ch) * RC + hr;
            if (h < p.H) {
              __nv_bfloat16* o = p.out + (((size_t)n * p.H + h) * WD) * MVALID + c;
#pragma unroll
              for (int w = 0; w < WD; ++w) o[(size_t)w * MVALID] = __float2bfloat16_rn(__uint_as_float(v[hr * WD + w]));
            }
          }
        }
      }
    }
  }
}

}  // namespace convsw

template <bool TRAIN, bool LINES = false, bool FP8 = false>
// `out`: NHWC map of the pooled output [N, H/2, 8, 128], box [64, 8, 8, 1] (one tile = 8 pooled rows); only <false> stores through it.
// FP8: a UINT8 map of the e4m3 output, box [128, 8, 8, 1]
static int launch_conv2_swap(const CUtensorMap& x, const CUtensorMap& w, const CUtensorMap& out, const convsw::Params& p, int num_sms,
                             cudaStream_t st) {
  static_assert(!(TRAIN && (LINES || FP8)), "line masks and e4m3 output exist in the inference epilogue only");
  auto kern = convsw::conv2_swap_kernel<TRAIN, LINES, FP8>;
  static bool attr = false;
  if (!attr) {
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, convsw::SMEM_BYTES));
    attr = true;
  }
  const int tiles = p.Nimg * p.tiles_per_img;
  const int grid = tiles < num_sms ? tiles : num_sms;
  kern<<<grid, convsw::NUM_THREADS, convsw::SMEM_BYTES, st>>>(x, w, out, p);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}

// the inference launch with LINES picked at run time: `lines` = a packed evaluation batch (crnn_forward_lines)
template <bool FP8 = false>
static int launch_conv2_swap_lines(bool lines, const CUtensorMap& x, const CUtensorMap& w, const CUtensorMap& out, const convsw::Params& p,
                                   int num_sms, cudaStream_t st) {
  if (lines) return launch_conv2_swap<false, true, FP8>(x, w, out, p, num_sms, st);
  return launch_conv2_swap<false, false, FP8>(x, w, out, p, num_sms, st);
}

template <int WD, int CB, int MVALID>
static int launch_conv_dgrad_swap(const CUtensorMap& x, const CUtensorMap& w, const convsw::DgradParams& p, int num_sms, cudaStream_t st) {
  auto kern = convsw::conv_dgrad_swap_kernel<WD, CB, MVALID>;
  static bool attr = false;
  if (!attr) {
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, convsw::SMEM_BYTES));
    attr = true;
  }
  const int tiles = p.Nimg * p.tiles_per_img;
  const int grid = tiles < num_sms ? tiles : num_sms;
  kern<<<grid, convsw::NUM_THREADS, convsw::SMEM_BYTES, st>>>(x, w, p);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
