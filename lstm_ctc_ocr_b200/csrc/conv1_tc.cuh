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
// builders (a ring of B_STAGES B tiles and a double-buffered input stage, so the build of tile i+1 overlaps the MMA +
// epilogue of tile i), warps 4..11 = two MMA warpgroups (accumulator rows 0..63 / 64..127 = row set 0 / 1).
//
// Epilogue, in registers: accumulator column group j (8 columns) is image row hl = j/4 of the set, columns 8(j%4) + 2(l%4) +
// {0,1} a w pair, and group j + 4 the image row below, so a thread holds whole 2x2 windows of its two channels f0 and f0 + 8.
// Pool, bias, ReLU and bf16 rounding happen on the fragment; one shuffle with lane l ^ 4 gives each lane an adjacent channel
// pair.  A warpgroup's pooled output (4 pooled rows x 16 x 64 channels = 8 KB) is one contiguous range of `out`: it is staged
// in the SWIZZLE_128B layout of the NHWC tensor map and leaves with one TMA store (rows past the image dropped by the map),
// while the warpgroup goes on to its next tile.  The two warpgroups run independently: each has its own double-buffered
// staging and its own issuing thread.
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
constexpr int B_STAGES = 2;                      // B tiles in flight between the builders and the MMA warpgroups
constexpr int IN_ROWS = 18, IN_STRIDE = 36;      // staged input: image rows h0-1 .. h0+16, columns -1 .. 32 (+2 pad)
constexpr int IN_BYTES = IN_ROWS * IN_STRIDE * 4;
constexpr int OUT_BYTES = 4 * 16 * 64 * 2;       // one warpgroup's pooled tile: [4 pooled rows][16][64 channels] bf16
constexpr int AM_BYTES = 4 * 16 * 64;            // its pool1 arg-max bytes (training)
constexpr int OFF_B = A_BYTES;
constexpr int OFF_OUT = OFF_B + B_STAGES * B_BYTES;   // [2 warpgroups][2 buffers] pooled tiles (1024-aligned: SWIZZLE_128B)
constexpr int OFF_AM = OFF_OUT + 4 * OUT_BYTES;       // [2 warpgroups][2 buffers] arg-max tiles, linear NHWC
constexpr int OFF_IN = OFF_AM + 4 * AM_BYTES;
constexpr int OFF_BAR = (OFF_IN + 2 * IN_BYTES + 15) / 16 * 16;
constexpr int SMEM_BYTES = OFF_BAR + 128 + 1024;
static_assert(OFF_OUT % 1024 == 0, "SWIZZLE_128B staging must be 1024-byte aligned");
static_assert(SMEM_BYTES <= 232448, "opt-in shared memory per block (227 KB)");

// K column k (0..31) of a patch: part = k / 10 (x: hi, lo, hi | w: hi, hi, lo), tap = k % 10; tap 9 and k >= 30 are zero padding
__device__ __forceinline__ uint32_t bf16_bits(float v) { return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(v)); }
__device__ __forceinline__ float bf16_back(uint32_t b) { return __uint_as_float(b << 16); }

struct Params {
  const void* data;         // images img0 .. img0+N-1: [N, W, 32] f32 or uint8 (the kernel's TIn)
  const float* wgt;         // HWIO [3,3,1,64]
  const float* bias;        // [64]
  uint8_t* argmax;          // TRAIN: window index (dy*2+dx) of the max, [N, W/2, 16, 64] (this launch's images)
  int N, W, tiles_per_img;  // tiles_per_img = ceil(W / 16)
  int img0;                 // image coordinate of the first image in the output map
  const int* line_w;        // LINES: [N] clamped line widths (this launch's images); input columns >= line_w read as zero and
                            // pooled rows >= line_w / 2 are stored as zero (packed evaluation, crnn_forward_lines)
};

// `tmO`: NHWC map of the whole pooled output [*, W/2, 16, 64] bf16, box [64, 16, 4, 1], SWIZZLE_128B
// TIn: float (the f32 data tensor) or uint8_t (pixel bytes, widened to the same f32 values when they are staged: common.cuh)
template <bool TRAIN, bool LINES = false, typename TIn = float>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv1_tc_kernel(const __grid_constant__ CUtensorMap tmO, const Params p) {
  using Px = Pixels4<TIn>;
  extern __shared__ uint8_t smem_raw[];
  // aligned by OFFSET (not by casting through an integer): the pointers stay in the shared address space -> LDS/STS, not LD/ST
  uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + OFF_B;
  float* s_in = reinterpret_cast<float*>(smem + OFF_IN);
  uint64_t* b_full = reinterpret_cast<uint64_t*>(smem + OFF_BAR);   // [B_STAGES]
  uint64_t* b_empty = b_full + B_STAGES;

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.N * p.tiles_per_img;

  if (warp_idx == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmO);
    for (int s = 0; s < B_STAGES; ++s) {
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
    auto fetch = [&](int tile, typename Px::Raw (&v)[2]) {
      const int n = tile / p.tiles_per_img;
      const int h0 = (tile - n * p.tiles_per_img) * 16;
      const int wl = LINES ? __ldg(p.line_w + n) : p.W;
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int e = bt + k * BUILD_THREADS;
        const int r = e >> 3, c4 = e & 7;
        const int gr = h0 - 1 + r;
        v[k] = Px::zero();
        if (e < IN_ROWS * 8 && gr >= 0 && gr < wl) v[k] = Px::load(static_cast<const TIn*>(p.data) + ((size_t)n * p.W + gr) * 32, c4);
      }
    };
    auto stash = [&](float* stg, const typename Px::Raw (&raw)[2]) {
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int e = bt + k * BUILD_THREADS;
        if (e < IN_ROWS * 8) {
          const float4 v = Px::f32(raw[k]);
          float* d = stg + (e >> 3) * IN_STRIDE + 1 + (e & 7) * 4;
          d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
        }
      }
    };
    for (int b = 0; b < 2; ++b)                               // zero halo columns of both stages, once
      if (bt < IN_ROWS) { s_in[b * IN_ROWS * IN_STRIDE + bt * IN_STRIDE] = 0.f; s_in[b * IN_ROWS * IN_STRIDE + bt * IN_STRIDE + 33] = 0.f; }
    typename Px::Raw pre[2];
    if (blockIdx.x < num_tiles) {
      fetch(blockIdx.x, pre);
      stash(s_in, pre);
    }
    int it = 0, st = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int si = it & 1;                                  // input stage
      float* stg = s_in + si * (IN_ROWS * IN_STRIDE);
      const int nxt = tile + gridDim.x;
      if (nxt < num_tiles) fetch(nxt, pre);
      asm volatile("bar.sync 2, %0;" ::"n"(BUILD_THREADS) : "memory");
      ptx::mbar_wait(&b_empty[st], ph ^ 1);                  // the MMAs that read this B buffer B_STAGES tiles ago have retired
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
      if (nxt < num_tiles) stash(s_in + (si ^ 1) * (IN_ROWS * IN_STRIDE), pre);
      if (++st == B_STAGES) { st = 0; ph ^= 1; }
    }
  } else {
    // ===================== MMA (accumulator rows wgi*64 .. = row set wgi) + register-side epilogue =====================
    const int wgi = (warp_idx >> 2) - 1;
    const int t = threadIdx.x & 127;
    const bool issuer = t == 0;                              // arrives on b_empty and issues the warpgroup's stores
    const int f0 = 16 * (t >> 5) + (lane >> 2);              // this thread's channels: f0 (registers 4j, 4j+1) and f0 + 8 (4j+2, 4j+3)
    const float bias0 = __ldg(p.bias + f0), bias8 = __ldg(p.bias + f0 + 8);
    const float nbias0 = -bias0, nbias8 = -bias8;
    const bool even = ((lane >> 2) & 1) == 0;                // lanes l and l ^ 4 hold channels f0 and f0 ^ 1
    const int ch = even ? f0 : f0 + 7;                       // first channel of the pair this lane stores
    const int Hp = p.W >> 1;
    uint8_t* stg_out = smem + OFF_OUT + wgi * 2 * OUT_BYTES;
    uint8_t* stg_am = smem + OFF_AM + wgi * 2 * AM_BYTES;
    int it = 0, st = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int nl = tile / p.tiles_per_img;
      const int h0 = (tile - nl * p.tiles_per_img) * 16;
      ptx::mbar_wait(&b_full[st], ph);
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
      if (issuer) ptx::mbar_arrive(&b_empty[st]);
      if (++st == B_STAGES) { st = 0; ph ^= 1; }

      // This tile's staging buffer was last read by the store issued two tiles ago; the issuer waited for that read before the
      // previous tile's barrier.
      uint8_t* so = stg_out + (it & 1) * OUT_BYTES;
      uint8_t* sa = stg_am + (it & 1) * AM_BYTES;
      const int hl_end = LINES ? (__ldg(p.line_w + nl) >> 1) - ((h0 >> 1) + 4 * wgi) : 4;   // pooled rows of this tile inside the line
#pragma unroll
      for (int pr = 0; pr < 4; ++pr) {                       // pooled row pr: image rows 2pr, 2pr+1 = column groups 8pr + i, 8pr + i + 4
#pragma unroll
        for (int ip = 0; ip < 4; ip += 2) {                  // pooled columns 4i + l%4 of i = ip, ip + 1
          uint32_t wv[2], wa[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int j = 8 * pr + ip + e;
            uint32_t v, a0 = 0, a8 = 0;                       // v: bf16 of channel f0 (low half) and f0 + 8 (high half)
            if (!TRAIN) {
              // relu(max4 + b) == max(max4, -b) + b exactly (the same FADD on the same operand, or (-b) + b = 0): two 3-input
              // maxima and one add instead of three maxima, an add and a max
              const float m0 = fmaxf(fmaxf(fmaxf(d[4 * j], d[4 * j + 1]), fmaxf(d[4 * j + 16], d[4 * j + 17])), nbias0);
              const float m8 = fmaxf(fmaxf(fmaxf(d[4 * j + 2], d[4 * j + 3]), fmaxf(d[4 * j + 18], d[4 * j + 19])), nbias8);
              v = ptx::pack_bf16x2(m0 + bias0, m8 + bias8);
            } else {
              // strict '>' in (dy, dx) row-major order keeps the FIRST maximum (tie-break of TF/torch max-pool gradients),
              // decided on the f32 accumulators like the SIMT kernel
              float b0 = d[4 * j], b8 = d[4 * j + 2];
              if (d[4 * j + 1] > b0) { b0 = d[4 * j + 1]; a0 = 1; }
              if (d[4 * j + 16] > b0) { b0 = d[4 * j + 16]; a0 = 2; }
              if (d[4 * j + 17] > b0) { b0 = d[4 * j + 17]; a0 = 3; }
              if (d[4 * j + 3] > b8) { b8 = d[4 * j + 3]; a8 = 1; }
              if (d[4 * j + 18] > b8) { b8 = d[4 * j + 18]; a8 = 2; }
              if (d[4 * j + 19] > b8) { b8 = d[4 * j + 19]; a8 = 3; }
              v = ptx::pack_bf16x2(fmaxf(b0 + bias0, 0.f), fmaxf(b8 + bias8, 0.f));
            }
            // exchange with lane l ^ 4 (value in the low half, arg-max above it) so that each lane holds an adjacent channel
            // pair: (f0, f0 + 1) or (f0 + 7, f0 + 8)
            const uint32_t s0 = (v & 0xFFFFu) | (a0 << 16), s8 = (v >> 16) | (a8 << 16);
            const uint32_t r = __shfl_xor_sync(0xffffffffu, even ? s8 : s0, 4);
            wv[e] = even ? ((s0 & 0xFFFFu) | (r << 16)) : ((r & 0xFFFFu) | (v & 0xFFFF0000u));
            if (TRAIN) wa[e] = even ? (a0 | ((r >> 16) << 8)) : ((r >> 16) | (a8 << 8));
            if (LINES && pr >= hl_end) wv[e] = 0u;
          }
          // Odd lanes store their two positions in the other order: in each store instruction the even lanes' rows (chunk
          // 2*warp) and the odd lanes' rows (chunk 2*warp + 1) are 4 rows apart, so the swizzled 16-B chunks of the warp are all
          // different and the 32 words land in 32 banks.
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const bool first = (k == 0) == even;              // this instruction stores position i = ip (else ip + 1)
            const int row = pr * 16 + 4 * ip + (first ? 0 : 4) + (lane & 3);   // pooled position in the tile: [4 rows][16]
            *reinterpret_cast<uint32_t*>(so + row * 128 + ((((ch >> 3) ^ row) & 7) << 4) + ((ch & 7) << 1)) = first ? wv[0] : wv[1];
            if (TRAIN) *reinterpret_cast<uint16_t*>(sa + row * 64 + ch) = (uint16_t)(first ? wa[0] : wa[1]);
          }
        }
      }
      ptx::fence_proxy_async_smem();
      if (issuer) ptx::bulk_wait_read_all();                 // the previous tile's store has read its buffer: free for the next tile
      ptx::bar_sync(3 + wgi, 128);
      const int hp0 = (h0 >> 1) + 4 * wgi;                   // first pooled row of this warpgroup's tile
      if (issuer && hp0 < Hp) {                              // W = 16k + 8: the second warpgroup's tile lies past the image end
        ptx::tma_store_4d(&tmO, so, 0, 0, hp0, p.img0 + nl);    // rows >= Hp are dropped by the map
        if (TRAIN) ptx::bulk_store_1d(p.argmax + ((size_t)nl * Hp + hp0) * (16 * 64), sa, (uint32_t)min(4, Hp - hp0) * (16 * 64));
        ptx::bulk_commit();
      }
    }
    if (issuer) ptx::bulk_wait_all();                        // the CTA's shared memory must outlive its last stores
  }
}

}  // namespace conv1tc

// `out`: NHWC map of the pooled output [*, W/2, 16, 64] bf16 with box [64, 16, 4, 1]; this launch writes images
// img0 .. img0+N-1 of it (`data` and `argmax` point at image img0).  `line_w` != nullptr: packed evaluation lines (inference only).
// `u8`: `data` holds uint8 pixels (crnn_*_u8), else f32.
template <typename TIn>
static int launch_conv1_tc_t(const CUtensorMap& out, const conv1tc::Params& p, int num_sms, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    CUDA_TRY(cudaFuncSetAttribute(conv1tc::conv1_tc_kernel<true, false, TIn>, cudaFuncAttributeMaxDynamicSharedMemorySize, conv1tc::SMEM_BYTES));
    CUDA_TRY(cudaFuncSetAttribute(conv1tc::conv1_tc_kernel<false, false, TIn>, cudaFuncAttributeMaxDynamicSharedMemorySize, conv1tc::SMEM_BYTES));
    CUDA_TRY(cudaFuncSetAttribute(conv1tc::conv1_tc_kernel<false, true, TIn>, cudaFuncAttributeMaxDynamicSharedMemorySize, conv1tc::SMEM_BYTES));
    attr = true;
  }
  const int tiles = p.N * p.tiles_per_img;
  const int grid = tiles < num_sms ? tiles : num_sms;
  if (p.line_w != nullptr) conv1tc::conv1_tc_kernel<false, true, TIn><<<grid, conv1tc::NUM_THREADS, conv1tc::SMEM_BYTES, st>>>(out, p);
  else if (p.argmax != nullptr) conv1tc::conv1_tc_kernel<true, false, TIn><<<grid, conv1tc::NUM_THREADS, conv1tc::SMEM_BYTES, st>>>(out, p);
  else conv1tc::conv1_tc_kernel<false, false, TIn><<<grid, conv1tc::NUM_THREADS, conv1tc::SMEM_BYTES, st>>>(out, p);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}

static int launch_conv1_tc(const CUtensorMap& out, const void* data, bool u8, const float* w, const float* b, int img0, uint8_t* argmax,
                           int N, int W, int num_sms, cudaStream_t st, const int* line_w = nullptr) {
  conv1tc::Params p;
  p.data = data; p.wgt = w; p.bias = b; p.argmax = argmax; p.N = N; p.W = W; p.tiles_per_img = (W + 15) / 16; p.img0 = img0;
  p.line_w = line_w;
  return u8 ? launch_conv1_tc_t<uint8_t>(out, p, num_sms, st) : launch_conv1_tc_t<float>(out, p, num_sms, st);
}
