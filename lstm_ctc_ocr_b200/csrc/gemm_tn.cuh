// "TN" wgmma GEMM for weight gradients:  D[M x N] += sum_k A[k][m] * B[k][n]
// Both operands are stored K-rows x channel-columns (channels contiguous) -- exactly how activations and their
// gradients already sit in HBM (NHWC / [rows, C]) -- so they are fed to the tensor core as MN-MAJOR operands
// (wgmma transpose flags set for A and B) without any transposition pass.
//
// smem tile per operand and stage: J blocks of [64 K-rows x 128 B] (64 channels), 128-byte swizzle as written by
// TMA; canonical MN-major layout ((8,n),(8,k)) : leading byte offset = 8192 B between 64-channel blocks,
// stride byte offset = 1024 B between 8-row K groups; one wgmma consumes 16 K-rows (= 2048 B advance).
//
// Roles (384 threads): warpgroup 0 = TMA producer (warp 0), warpgroups 1 and 2 = MMA (M rows 0..63 / 64..127 = A block 0 / 1)
// and epilogue (accumulators staged in shared memory, thread = one output row, two warps per 32-row quadrant).
//
// Split-K persistent scheduler: work item = (output tile, K-chunk); the f32 tile is reduced into global memory with
// red.global.add.f32 (the gradient buffer is zeroed once per step).
//
// A modes: TN_PLAIN (2-D maps, K = matrix rows) and TN_CONV (K = output positions of a 3x3 SAME conv; the A box is
// the NHWC activation at tap-shifted coordinates, TMA OOB zero-fill supplies the padding; B = NHWC output gradient).
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace gemm_tn {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;                 // K rows per stage
constexpr int NUM_THREADS = 384;
constexpr int MAX_SMEM = 232448;
constexpr int BLK_BYTES = BLOCK_K * 128;    // one [64 x 64ch] block = 8 KB

enum AMode { TN_PLAIN = 0, TN_CONV = 1 };

struct Params {
  int num_m_tiles, num_n_tiles, num_taps;   // output tiles = taps x m x n
  int k_blocks_total;                        // K extent in 64-row blocks (TN_CONV: pairs of 32-row sub-boxes)
  int k_splits;                              // work items per output tile
  int M, N;                                  // valid output rows / cols
  // TN_CONV geometry
  int sb_per_img, bh, Wd, H, Nimg, Cin;
  int merged, kb_per_img;                    // TN_CONV: 64-position boxes (2*bh rows) when H % (2*bh) == 0
  int tap_pack_n;                            // TN_CONV with Cin == 64, operands SWAPPED (conv2 weight gradient): A = the output gradient
                                             // (M = Cout), B = the activation with FOUR tap-shifted 64-channel boxes per 256-column N tile
                                             // (columns = (tap, ci)); N = 256 restores the MMA rate the Cout = 128 N tile halves.  The
                                             // accumulator is written transposed: out[(tap*64 + ci) * ldo + co]
  int a_row_shift;                           // TN_PLAIN: A rows are read at k + a_row_shift (conv5's second tap)
  // output
  float* out;
  long long ldo;                             // row stride of out (elements)
  long long tap_stride;                      // TN_CONV: elements between taps (Cin*Cout)
  int lstm_cols;                             // != 0: output columns are permuted LSTM gate columns (upc = 32), two directions
  long long dir_stride;                      // elements between the two directions' matrices (lstm_cols)
  int out_row_offset;                        // added to the output row (LSTM: h rows start at 512)
};

// MN-major, 128B swizzle: LBO = 8192 B (between 64-element MN blocks), SBO = 1024 B (between 8-row K groups)
__device__ __forceinline__ uint64_t make_desc_mn_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(BLK_BYTES >> 4) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

template <int BLOCK_N, int STAGES>
struct Smem {
  static constexpr int A_STAGE = (BLOCK_M / 64) * BLK_BYTES;
  static constexpr int B_STAGE = (BLOCK_N / 64) * BLK_BYTES;
  static constexpr int ACC_BYTES = BLOCK_M * BLOCK_N * 4;
  static constexpr int FIT = (MAX_SMEM - ACC_BYTES - 256 - 1024) / (A_STAGE + B_STAGE);
  static constexpr int S = STAGES < FIT ? STAGES : FIT;
  static constexpr int ACC_OFFSET = S * (A_STAGE + B_STAGE);
  static constexpr int BAR_OFFSET = ACC_OFFSET + ACC_BYTES;
  static constexpr int BYTES = BAR_OFFSET + 256 + 1024;
};

template <int BLOCK_N, int AMODE, int STAGES>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const Params p) {
  using SM = Smem<BLOCK_N, STAGES>;
  constexpr int A_STAGE = SM::A_STAGE, B_STAGE = SM::B_STAGE, STG = SM::S;
  constexpr int JA = BLOCK_M / 64, JB = BLOCK_N / 64;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STG * A_STAGE;
  float* acc_tile = reinterpret_cast<float*>(smem + SM::ACC_OFFSET);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + SM::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STG;

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles = p.num_taps * p.num_m_tiles * p.num_n_tiles;
  const int num_items = tiles * p.k_splits;
  const int kb_per_split = (p.k_blocks_total + p.k_splits - 1) / p.k_splits;

  if (warp_idx == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmB);
    for (int s = 0; s < STG; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], 2); }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  // work item -> (tap, m_blk, n_blk, [kb0, kb1)) ; K-split is the slowest index so concurrently running CTAs work
  // on the same K-chunk of different tiles (operand reuse in L2)
  auto decode = [&](int item, int& tap, int& m_blk, int& n_blk, int& kb0, int& kb1) {
    const int split = item / tiles;
    int t = item - split * tiles;
    n_blk = t % p.num_n_tiles; t /= p.num_n_tiles;
    m_blk = t % p.num_m_tiles; tap = t / p.num_m_tiles;
    kb0 = split * kb_per_split;
    kb1 = min(kb0 + kb_per_split, p.k_blocks_total);
  };

  if (warp_idx < 4) {
    // one lane per 64-channel operand block (JA blocks of A, JB blocks of B); lane 0 also arms the transaction count
    ptx::setmaxnreg_dec<40>();
    if (warp_idx == 0 && lane < JA + JB) {
      const bool isA = lane < JA;
      const int j = isA ? lane : lane - JA;
      int stage = 0; uint32_t phase = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        int tap, m_blk, n_blk, kb0, kb1;
        decode(item, tap, m_blk, n_blk, kb0, kb1);
        int r = tap / 3, s = tap - 3 * r;
        int ccol = isA ? (m_blk * BLOCK_M + 64 * j) : (n_blk * BLOCK_N + 64 * j);
        bool shifted = isA;                                 // which operand's boxes carry the (r-1, s-1) tap shift
        if (AMODE == TN_CONV && p.tap_pack_n) {            // B block j of tile n_blk is tap 4*n_blk + j (taps >= 9: columns masked)
          shifted = !isA;
          if (!isA) { const int tp = min(4 * n_blk + j, 8); r = tp / 3; s = tp - 3 * r; ccol = 0; }
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          if (lane == 0) ptx::mbar_arrive_expect_tx(&full_bar[stage], A_STAGE + B_STAGE);
          uint8_t* dst = (isA ? smem_a + stage * A_STAGE : smem_b + stage * B_STAGE) + j * BLK_BYTES;
          const CUtensorMap* tm = isA ? &tmA : &tmB;
          if (AMODE == TN_PLAIN) {
            ptx::tma_load_2d(tm, &full_bar[stage], dst, ccol, kb * BLOCK_K + (isA ? p.a_row_shift : 0));
          } else if (p.merged) {
            // 64 consecutive positions = 2*bh rows of one image in one box
            const int n = kb / p.kb_per_img;
            const int h0 = (kb - n * p.kb_per_img) * 2 * p.bh;
            ptx::tma_load_4d(tm, &full_bar[stage], dst, ccol, shifted ? s - 1 : 0, h0 + (shifted ? r - 1 : 0), n);
          } else {
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              const int g = kb * 2 + half;                     // 32-position sub-box index
              const int n = g / p.sb_per_img;
              const int h0 = (g - n * p.sb_per_img) * p.bh;
              ptx::tma_load_4d(tm, &full_bar[stage], dst + half * 4096, ccol, shifted ? s - 1 : 0, h0 + (shifted ? r - 1 : 0), n);
            }
          }
          if (++stage == STG) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<232>();
    const int wgi = (warp_idx >> 2) - 1;             // M rows wgi*64 .. = A block wgi
    const int chalf = (warp_idx - 4) >> 2;           // warps 4..7 drain columns [0, N/2), warps 8..11 [N/2, N)
    const bool arriver = (warp_idx & 3) == 0 && lane == 0;
    int stage = 0; uint32_t phase = 0;
    const int q = warp_idx & 3;
    const int row = q * 32 + lane;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      int tap, m_blk, n_blk, kb0, kb1;
      decode(item, tap, m_blk, n_blk, kb0, kb1);
      float d[BLOCK_N / 2];
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) d[i] = 0.f;     // an empty K chunk reduces zeros
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        ptx::mbar_wait(&full_bar[stage], phase);
        const uint64_t a_desc = make_desc_mn_sw128(ptx::smem_u32(smem_a + stage * A_STAGE + wgi * BLK_BYTES));
        const uint64_t b_desc = make_desc_mn_sw128(ptx::smem_u32(smem_b + stage * B_STAGE));
        wg::fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / 16; ++k)     // 16 K-rows = 2048 B -> +128 in the (addr >> 4) field
          wg::mma_bf16<BLOCK_N, 1>(d, a_desc + 128 * k, b_desc + 128 * k, 1u);
        wg::commit();
        wg::wait<1>();
        if (prev >= 0 && arriver) ptx::mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STG) { stage = 0; phase ^= 1; }
      }
      wg::wait<0>();
      wg::fence_operand(d);
      if (prev >= 0 && arriver) ptx::mbar_arrive(&empty_bar[prev]);
      ptx::bar_sync(1, 256);
      ptx::acc_store<BLOCK_N, BLOCK_N>(acc_tile, d, wgi * 64);
      ptx::bar_sync(1, 256);
      const int m = m_blk * BLOCK_M + row;
      const bool okm = (m < p.M) && (kb1 > kb0);
      float* orow = p.out + (long long)tap * p.tap_stride + (long long)(m + p.out_row_offset) * p.ldo;
#pragma unroll 1
      for (int c0 = chalf * (BLOCK_N / 2); c0 < (chalf + 1) * (BLOCK_N / 2); c0 += 32) {
        uint32_t v[32];
        ptx::acc_ld<BLOCK_N, 32>(acc_tile, row, c0, v);
        if (AMODE == TN_CONV && p.tap_pack_n) {
          // swapped operands: row = output channel co, column = (tap, ci).  Written transposed into the HWIO gradient
          // out[(tap*64 + ci) * ldo + co]; the lanes of a warp are consecutive co -> one 128-byte segment per instruction
          const int tp = 4 * n_blk + (c0 >> 6), ci0 = c0 & 63;
          if (okm && tp < 9) {
            float* dst = p.out + (long long)(tp * 64 + ci0) * p.ldo + m;
#pragma unroll
            for (int i = 0; i < 32; ++i) atomicAdd(dst + (long long)i * p.ldo, __uint_as_float(v[i]));
          }
          continue;
        }
        const int ncol = n_blk * BLOCK_N + c0;
        if (okm && ncol < p.N) {
          float* dst;
          if (p.lstm_cols) {
            // permuted gate column pc = dir*1024 + (u/32)*128 + g*32 + u%32  ->  TF column g*256 + u
            const int dir = ncol >> 10, pc = ncol & 1023;
            const int g = (pc & 127) >> 5, ub = pc >> 7;
            dst = orow + (long long)dir * p.dir_stride + g * 256 + ub * 32;
          } else {
            dst = orow + ncol;
          }
          // split-K reduction straight into the gradient tensor: 128-bit vector reds (a quarter of the L2 atomic transactions of
          // scalar atomicAdd; every destination is 16-byte aligned: tensor offsets, row strides and column starts are multiples of 4)
#pragma unroll
          for (int i = 0; i < 32; i += 4)
            ptx::red_add_v4_f32(dst + i, __uint_as_float(v[i]), __uint_as_float(v[i + 1]), __uint_as_float(v[i + 2]), __uint_as_float(v[i + 3]));
        }
      }
    }
  }
}



}  // namespace gemm_tn
